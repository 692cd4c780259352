// TMOT / JDE association in native host code (SURVEY 8f rank 4): the matching distances of tmot/matching.py:28-109
// (linear_assignment over lap.lapjv, ious / iou_distance, embedding_distance, fuse_motion) and the JDETracker loop of
// tmot/multitracker.py:13-398 (STrack life cycle, smoothed embeddings, three association rounds, lost / removed
// bookkeeping, duplicate removal).  State is float64 like the reference; embeddings are float32 like the arrays the
// reference driver feeds (obj_detect_tracking_multi_queuer_tmot.py:545-566).  The embedding distance of every frame is
// one tensor-core GEMM (b2_distance_matrix, squared euclidean, then sqrt) unless the caller installs a cost function
// (tests install the CPU oracle there; there is no built-in CPU path).
//
// Third-party pieces the reference calls that are NOT under /root/reference, restated from their published algorithms:
//   lap.lapjv(cost, extend_cost=True, cost_limit=L)  (lap 0.4.0, `import lap  # 0.4.0` matching.py:4): the cost matrix is
//     embedded in an (nr+nc)^2 matrix filled with L/2, zeros in the lower-right block, solved as a square assignment;
//     rows/columns assigned to the padding are reported unmatched.  Solved here with the SciPy-exact solver of assoc.h;
//     the optimum is unique for tie-free costs (which real-valued distances are), lap's own tie order is unpinned.
//   cython_bbox.bbox_overlaps  (matching.py:6): IoU with the +1 pixel convention of py-faster-rcnn's bbox.pyx.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <limits>
#include <memory>
#include <set>
#include <vector>

#include "../../include/b200det.h"
#include "common.h"

#include "assoc.h"

namespace b2 {
namespace {

enum { kNew = 0, kTracked = 1, kLost = 2, kRemoved = 3 };   // tmot/basetrack.py:5-9

// lap.lapjv(cost, extend_cost=True, cost_limit=limit): x[nr], y[nc] (-1 = unmatched); returns the matched cost sum.
int lapjv_limit(const double* cost, int nr, int nc, double limit, std::vector<int>& x, std::vector<int>& y, double* opt) {
  x.assign(nr, -1);
  y.assign(nc, -1);
  if (opt) *opt = 0;
  if (nr == 0 || nc == 0) return 0;
  const int n = nr + nc;
  std::vector<double> ext(static_cast<size_t>(n) * n, limit / 2.0);
  for (int i = nr; i < n; ++i)
    for (int j = nc; j < n; ++j) ext[static_cast<size_t>(i) * n + j] = 0.0;
  for (int i = 0; i < nr; ++i)
    for (int j = 0; j < nc; ++j) {
      const double c = cost[static_cast<size_t>(i) * nc + j];
      if (c != c) return -1;
      ext[static_cast<size_t>(i) * n + j] = c;
    }
  std::vector<int> rows, cols;
  if (lsap(n, n, ext.data(), rows, cols) != 0) return -1;
  double s = 0;
  for (size_t k = 0; k < rows.size(); ++k) {
    const int r = rows[k], c = cols[k];
    if (r < nr && c < nc) {
      x[r] = c;
      y[c] = r;
      s += cost[static_cast<size_t>(r) * nc + c];
    }
  }
  if (opt) *opt = s;
  return 0;
}

// matching.py:41-77: 1 - IoU(+1 convention) of tlbr boxes
void iou_distance(const double* a, int na, const double* b, int nb, double* out) {
  for (int i = 0; i < na; ++i) {
    const double* p = a + 4 * i;
    const double area_p = (p[2] - p[0] + 1) * (p[3] - p[1] + 1);
    for (int j = 0; j < nb; ++j) {
      const double* q = b + 4 * j;
      double iou = 0;
      const double iw = std::min(p[2], q[2]) - std::max(p[0], q[0]) + 1;
      if (iw > 0) {
        const double ih = std::min(p[3], q[3]) - std::max(p[1], q[1]) + 1;
        if (ih > 0) {
          const double area_q = (q[2] - q[0] + 1) * (q[3] - q[1] + 1);
          iou = iw * ih / (area_p + area_q - iw * ih);
        }
      }
      out[static_cast<size_t>(i) * nb + j] = 1.0 - iou;
    }
  }
}

// squared Mahalanobis distance on the first `dims` (2 or 4) measurement dimensions (tmot/kalman_filter.py:230-277)
bool gating_distance(const double mean[8], const double cov[64], const double* zs, int n, int dims, double* out) {
  double pm[4], pc[16];
  kf_project(mean, cov, pm, pc);
  if (dims == 4) return kf_gating(mean, cov, zs, n, out);
  // 2x2 Cholesky of the position block
  const double a = pc[0], b = pc[4], c = pc[5];
  if (!(a > 0)) return false;
  const double l00 = sqrt(a), l10 = b / l00;
  const double d = c - l10 * l10;
  if (!(d > 0)) return false;
  const double l11 = sqrt(d);
  for (int k = 0; k < n; ++k) {
    const double y0 = (zs[4 * k] - pm[0]) / l00;
    const double y1 = (zs[4 * k + 1] - pm[1] - l10 * y0) / l11;
    out[k] = y0 * y0 + y1 * y1;
  }
  return true;
}

// matching.py:97-109
bool fuse_motion(const double* means, const double* covs, int T, const double* xyah, int N, double* cost, int only_position,
                 double lambda) {
  if (T == 0 || N == 0) return true;
  const double thr = only_position ? 5.9915 : kChi2Inv95_4;
  std::vector<double> g(N);
  const double inf = std::numeric_limits<double>::infinity();
  for (int r = 0; r < T; ++r) {
    if (!gating_distance(means + 8 * r, covs + 64 * r, xyah, N, only_position ? 2 : 4, g.data())) return false;
    double* row = cost + static_cast<size_t>(r) * N;
    for (int c = 0; c < N; ++c) {
      if (g[c] > thr) row[c] = inf;
      row[c] = lambda * row[c] + (1 - lambda) * g[c];
    }
  }
  return true;
}

void normalize_f32(std::vector<float>& v) {   // feat /= np.linalg.norm(feat)  (float32 arrays)
  double ss = 0;
  for (float x : v) ss += static_cast<double>(x) * x;
  const float nrm = static_cast<float>(sqrt(ss));
  for (float& x : v) x = x / nrm;
}

struct STrack {   // multitracker.py:13-174
  double tlwh0[4];                 // _tlwh
  double mean[8], cov[64];
  bool has_mean = false, is_activated = false;
  double score = 0;
  int tracklet_len = 0, track_id = 0, state = kNew, frame_id = 0, start_frame = 0;
  std::vector<float> smooth_feat, curr_feat;
  double cur_det_tlwh[4];
  double cur_det_conf = 0;

  // __init__ -> update_features (:15-44): smooth_feat is None, so curr_feat and smooth_feat are the SAME array and both
  // in-place normalisations (:37 and :44) land on it.
  void init_features(const float* feat, int D) {
    curr_feat.assign(feat, feat + D);
    normalize_f32(curr_feat);
    normalize_f32(curr_feat);
    smooth_feat = curr_feat;
  }
  // update_features on a live track (:36-44): float32 arrays, the Python-float weights act as float32 scalars
  void update_features(const std::vector<float>& feat_in, double alpha) {
    curr_feat = feat_in;
    normalize_f32(curr_feat);
    const float a = static_cast<float>(alpha), b = static_cast<float>(1 - alpha);
    for (size_t i = 0; i < curr_feat.size(); ++i) {
      const float p = a * smooth_feat[i], q = b * curr_feat[i];
      smooth_feat[i] = p + q;
    }
    normalize_f32(smooth_feat);
  }
  void tlwh(double out[4]) const {   // :121-132
    if (!has_mean) {
      memcpy(out, tlwh0, sizeof(double) * 4);
      return;
    }
    out[2] = mean[2] * mean[3];
    out[3] = mean[3];
    out[0] = mean[0] - out[2] / 2;
    out[1] = mean[1] - out[3] / 2;
  }
  void tlbr(double out[4]) const {   // :134-142
    tlwh(out);
    out[2] += out[0];
    out[3] += out[1];
  }
  void xyah(double out[4]) const {   // :144-156
    tlwh(out);
    out[0] += out[2] / 2;
    out[1] += out[3] / 2;
    out[2] /= out[3];
  }
};

typedef std::shared_ptr<STrack> TrackPtr;
typedef std::vector<TrackPtr> TrackList;

TrackList joint_stracks(const TrackList& a, const TrackList& b) {   // :360-371
  std::set<int> exists;
  TrackList res;
  for (const TrackPtr& t : a) {
    exists.insert(t->track_id);
    res.push_back(t);
  }
  for (const TrackPtr& t : b)
    if (exists.insert(t->track_id).second) res.push_back(t);
  return res;
}

// :373-381 (a dict keyed by track id: insertion order, a later duplicate id replaces the value in place)
TrackList dict_by_id(const TrackList& a) {
  TrackList res;
  for (const TrackPtr& t : a) {
    bool found = false;
    for (TrackPtr& r : res)
      if (r->track_id == t->track_id) {
        r = t;
        found = true;
        break;
      }
    if (!found) res.push_back(t);
  }
  return res;
}

}  // namespace
}  // namespace b2

using namespace b2;

struct b2_jde {
  int device = 0, precision = 1, feat_dim = 0;
  double det_thresh = 0, max_frame_lost = 0, emb_max_dist = 0.7, iou_max_dist1 = 0.8, iou_max_dist2 = 0.9, alpha = 0.9;
  int frame_id = 0;
  std::shared_ptr<int> id_counter;          // BaseTrack._count is a class attribute: shared by every tracker (basetrack.py:13,34-37)
  b2_appearance_cost_fn cost_fn = nullptr;
  void* cost_user = nullptr;
  TrackList tracked, lost;
  std::set<int> removed_ids;                // self.removed_stracks is only ever used through its track ids (sub_stracks)
  TrackList output;
};

namespace {

TrackList sub_by_ids(const TrackList& a, const std::set<int>& ids) {
  TrackList res;
  for (const TrackPtr& t : dict_by_id(a))
    if (!ids.count(t->track_id)) res.push_back(t);
  return res;
}

TrackList sub_stracks(const TrackList& a, const TrackList& b) {
  std::set<int> ids;
  for (const TrackPtr& t : b) ids.insert(t->track_id);
  TrackList res;
  for (const TrackPtr& t : dict_by_id(a))
    if (!ids.count(t->track_id)) res.push_back(t);
  return res;
}

// matching.py:28-38
int assign(const std::vector<double>& cost, int nr, int nc, double thresh, std::vector<std::pair<int, int>>& matches,
           std::vector<int>& ua, std::vector<int>& ub) {
  matches.clear();
  ua.clear();
  ub.clear();
  if (nr == 0 || nc == 0) {
    for (int i = 0; i < nr; ++i) ua.push_back(i);
    for (int j = 0; j < nc; ++j) ub.push_back(j);
    return 0;
  }
  std::vector<int> x, y;
  B2_CHECK(lapjv_limit(cost.data(), nr, nc, thresh, x, y, nullptr) == 0, "jde: assignment failed (NaN cost)");
  for (int i = 0; i < nr; ++i) {
    if (x[i] >= 0) matches.push_back(std::make_pair(i, x[i]));
    else ua.push_back(i);
  }
  for (int j = 0; j < nc; ++j)
    if (y[j] < 0) ub.push_back(j);
  return 0;
}

void iou_cost(const TrackList& a, const TrackList& b, std::vector<double>& cost) {
  std::vector<double> ba(a.size() * 4), bb(b.size() * 4);
  for (size_t i = 0; i < a.size(); ++i) a[i]->tlbr(&ba[4 * i]);
  for (size_t j = 0; j < b.size(); ++j) b[j]->tlbr(&bb[4 * j]);
  cost.resize(a.size() * b.size());
  iou_distance(ba.data(), static_cast<int>(a.size()), bb.data(), static_cast<int>(b.size()), cost.data());
}

// np.maximum(0, d): a NaN distance stays NaN (std::max(0.0, NaN) is 0, a perfect match), and the assignment refuses it
double clamp0(double d) { return d < 0.0 ? 0.0 : d; }

int embedding_cost(b2_jde* t, const TrackList& pool, const TrackList& dets, std::vector<double>& cost) {   // matching.py:80-94
  const int T = static_cast<int>(pool.size()), N = static_cast<int>(dets.size()), D = t->feat_dim;
  cost.assign(static_cast<size_t>(T) * N, 0.0);
  if (T == 0 || N == 0) return 0;
  std::vector<float> a(static_cast<size_t>(T) * D), b(static_cast<size_t>(N) * D), c32(static_cast<size_t>(T) * N);
  for (int r = 0; r < T; ++r) memcpy(&a[static_cast<size_t>(r) * D], pool[r]->smooth_feat.data(), sizeof(float) * D);
  for (int c = 0; c < N; ++c) memcpy(&b[static_cast<size_t>(c) * D], dets[c]->curr_feat.data(), sizeof(float) * D);
  if (t->cost_fn) {
    std::vector<int32_t> seg(T + 1);
    for (int r = 0; r <= T; ++r) seg[r] = r;
    if (t->cost_fn(t->cost_user, a.data(), seg.data(), T, b.data(), N, D, c32.data()) != 0) return -1;
    for (size_t i = 0; i < c32.size(); ++i) cost[i] = clamp0(static_cast<double>(c32[i]));
  } else {
    if (b2_distance_matrix(t->device, a.data(), T, b.data(), N, D, 1, t->precision, c32.data()) != 0) return -1;
    for (size_t i = 0; i < c32.size(); ++i) cost[i] = sqrt(clamp0(static_cast<double>(c32[i])));
  }
  return 0;
}

int track_update(STrack& tr, const STrack& det, int frame_id, double alpha) {   // :95-118
  tr.frame_id = frame_id;
  tr.tracklet_len += 1;
  double z[4];
  det.xyah(z);
  B2_CHECK(kf_update(tr.mean, tr.cov, z), "jde: innovation covariance not positive definite");
  tr.state = kTracked;
  tr.is_activated = true;
  tr.score = det.score;
  tr.update_features(det.curr_feat, alpha);
  memcpy(tr.cur_det_tlwh, det.cur_det_tlwh, sizeof(double) * 4);
  tr.cur_det_conf = det.cur_det_conf;
  return 0;
}

int track_reactivate(STrack& tr, const STrack& det, int frame_id, double alpha) {   // :78-93
  double z[4];
  det.xyah(z);
  B2_CHECK(kf_update(tr.mean, tr.cov, z), "jde: innovation covariance not positive definite");
  tr.update_features(det.curr_feat, alpha);
  tr.tracklet_len = 0;
  tr.state = kTracked;
  tr.is_activated = true;
  tr.frame_id = frame_id;
  memcpy(tr.cur_det_tlwh, det.cur_det_tlwh, sizeof(double) * 4);
  tr.cur_det_conf = det.cur_det_conf;
  return 0;
}

}  // namespace

extern "C" {

int b2_lapjv(const double* cost, int nr, int nc, double cost_limit, int32_t* x, int32_t* y, double* opt) {
  B2_CHECK(nr >= 0 && nc >= 0 && (nr == 0 || nc == 0 || cost), "b2_lapjv: bad argument");
  std::vector<int> xs, ys;
  B2_CHECK(lapjv_limit(cost, nr, nc, cost_limit, xs, ys, opt) == 0, "b2_lapjv: NaN in the cost matrix");
  for (int i = 0; i < nr; ++i) x[i] = xs[i];
  for (int j = 0; j < nc; ++j) y[j] = ys[j];
  return 0;
}

int b2_tmot_iou_distance(const double* atlbr, int na, const double* btlbr, int nb, double* out) {
  B2_CHECK(na >= 0 && nb >= 0 && (na * nb == 0 || (atlbr && btlbr && out)), "b2_tmot_iou_distance: bad argument");
  iou_distance(atlbr, na, btlbr, nb, out);
  return 0;
}

int b2_tmot_fuse_motion(const double* means, const double* covs, int T, const double* xyah, int N, double* cost,
                        int only_position, double lambda) {
  B2_CHECK(T >= 0 && N >= 0 && (T * N == 0 || (means && covs && xyah && cost)), "b2_tmot_fuse_motion: bad argument");
  B2_CHECK(fuse_motion(means, covs, T, xyah, N, cost, only_position, lambda),
           "b2_tmot_fuse_motion: projected covariance not positive definite");
  return 0;
}

int b2_tmot_embedding_distance(int device, const float* track_feats, int T, const float* det_feats, int N, int D,
                               int precision, double* out) {
  B2_CHECK(T >= 0 && N >= 0 && D > 0, "b2_tmot_embedding_distance: bad argument");
  if (T == 0 || N == 0) return 0;
  B2_CHECK(track_feats && det_feats && out, "b2_tmot_embedding_distance: null argument");
  std::vector<float> c32(static_cast<size_t>(T) * N);
  if (b2_distance_matrix(device, track_feats, T, det_feats, N, D, 1, precision, c32.data()) != 0) return -1;
  for (size_t i = 0; i < c32.size(); ++i) out[i] = sqrt(clamp0(static_cast<double>(c32[i])));
  return 0;
}

int b2_jde_create(b2_jde** out, int device, double conf_thres, double track_max_second_lost, double emb_max_dist,
                  double iou_max_dist1, double iou_max_dist2, double emb_smooth_alpha, double frame_gap, double frame_rate,
                  int feat_dim, int precision, b2_jde* share_ids_with) {
  B2_CHECK(out, "b2_jde_create: null argument");
  *out = nullptr;
  B2_CHECK(feat_dim > 0 && frame_gap > 0, "b2_jde_create: bad parameters");
  b2_jde* t = new b2_jde();
  t->device = device;
  t->precision = precision;
  t->feat_dim = feat_dim;
  t->det_thresh = conf_thres;
  t->max_frame_lost = track_max_second_lost * frame_rate / frame_gap;   // multitracker.py:193
  t->emb_max_dist = emb_max_dist;
  t->iou_max_dist1 = iou_max_dist1;
  t->iou_max_dist2 = iou_max_dist2;
  t->alpha = emb_smooth_alpha;
  t->id_counter = share_ids_with ? share_ids_with->id_counter : std::make_shared<int>(0);
  *out = t;
  return 0;
}

void b2_jde_destroy(b2_jde* t) { delete t; }

int b2_jde_set_cost_fn(b2_jde* t, b2_appearance_cost_fn fn, void* user) {
  B2_CHECK(t, "b2_jde_set_cost_fn: null tracker");
  t->cost_fn = fn;
  t->cost_user = user;
  return 0;
}

int b2_jde_reset(b2_jde* t) {   // multitracker.py:206-215 (also zeroes the shared id counter, as the reference does)
  B2_CHECK(t, "b2_jde_reset: null tracker");
  t->tracked.clear();
  t->lost.clear();
  t->removed_ids.clear();
  t->output.clear();
  t->frame_id = 0;
  *t->id_counter = 0;
  return 0;
}

int b2_jde_reset_ids(b2_jde* t) {   // BaseTrack._count = 0 alone (multitracker.py:215), for a reset() of a group member without state
  B2_CHECK(t, "b2_jde_reset_ids: null tracker");
  *t->id_counter = 0;
  return 0;
}

int b2_jde_update(b2_jde* t, const double* tlwh, const double* conf, const float* features, int n) {   // :217-358
  B2_CHECK(t && (n == 0 || (tlwh && conf && features)), "b2_jde_update: null argument");
  const int D = t->feat_dim;
  t->frame_id += 1;
  TrackList activated, refind, lost_new, removed_new;
  TrackList dets(n);
  for (int i = 0; i < n; ++i) {
    dets[i] = std::make_shared<STrack>();
    STrack& d = *dets[i];
    memcpy(d.tlwh0, tlwh + 4 * i, sizeof(double) * 4);
    memcpy(d.cur_det_tlwh, tlwh + 4 * i, sizeof(double) * 4);
    d.score = conf[i];
    d.cur_det_conf = conf[i];
    d.init_features(features + static_cast<size_t>(i) * D, D);
  }
  TrackList unconfirmed, tracked;
  for (const TrackPtr& tr : t->tracked) (tr->is_activated ? tracked : unconfirmed).push_back(tr);

  // ---- step 2: first association, embedding distance fused with the Kalman gate ----
  TrackList pool = joint_stracks(tracked, t->lost);
  for (const TrackPtr& tr : pool) {   // STrack.multi_predict :52-63
    if (tr->state != kTracked) tr->mean[7] = 0;
    kf_predict_fp_ft(tr->mean, tr->cov);
  }
  std::vector<double> cost;
  if (embedding_cost(t, pool, dets, cost)) return -1;
  {
    const int T = static_cast<int>(pool.size());
    std::vector<double> means(static_cast<size_t>(T) * 8), covs(static_cast<size_t>(T) * 64), zs(static_cast<size_t>(n) * 4);
    for (int r = 0; r < T; ++r) {
      memcpy(&means[8 * r], pool[r]->mean, sizeof(double) * 8);
      memcpy(&covs[64 * r], pool[r]->cov, sizeof(double) * 64);
    }
    for (int c = 0; c < n; ++c) dets[c]->xyah(&zs[4 * c]);
    B2_CHECK(fuse_motion(means.data(), covs.data(), T, zs.data(), n, cost.data(), 0, 0.98),
             "jde: projected covariance not positive definite");
  }
  std::vector<std::pair<int, int>> matches;
  std::vector<int> u_track, u_det;
  if (assign(cost, static_cast<int>(pool.size()), n, t->emb_max_dist, matches, u_track, u_det)) return -1;
  for (const auto& m : matches) {
    STrack& tr = *pool[m.first];
    if (tr.state == kTracked) {
      if (track_update(tr, *dets[m.second], t->frame_id, t->alpha)) return -1;
      activated.push_back(pool[m.first]);
    } else {
      if (track_reactivate(tr, *dets[m.second], t->frame_id, t->alpha)) return -1;
      refind.push_back(pool[m.first]);
    }
  }

  // ---- step 3: second association, IoU ----
  TrackList dets2, r_tracked;
  for (int i : u_det) dets2.push_back(dets[i]);
  for (int i : u_track)
    if (pool[i]->state == kTracked) r_tracked.push_back(pool[i]);
  iou_cost(r_tracked, dets2, cost);
  if (assign(cost, static_cast<int>(r_tracked.size()), static_cast<int>(dets2.size()), t->iou_max_dist1, matches, u_track, u_det))
    return -1;
  for (const auto& m : matches) {
    STrack& tr = *r_tracked[m.first];
    if (tr.state == kTracked) {
      if (track_update(tr, *dets2[m.second], t->frame_id, t->alpha)) return -1;
      activated.push_back(r_tracked[m.first]);
    } else {
      if (track_reactivate(tr, *dets2[m.second], t->frame_id, t->alpha)) return -1;
      refind.push_back(r_tracked[m.first]);
    }
  }
  for (int i : u_track) {
    STrack& tr = *r_tracked[i];
    if (tr.state != kLost) {
      tr.state = kLost;
      lost_new.push_back(r_tracked[i]);
    }
  }

  // ---- unconfirmed tracks (one beginning frame so far), IoU ----
  TrackList dets3;
  for (int i : u_det) dets3.push_back(dets2[i]);
  iou_cost(unconfirmed, dets3, cost);
  std::vector<int> u_unconf;
  if (assign(cost, static_cast<int>(unconfirmed.size()), static_cast<int>(dets3.size()), t->iou_max_dist2, matches, u_unconf, u_det))
    return -1;
  for (const auto& m : matches) {
    if (track_update(*unconfirmed[m.first], *dets3[m.second], t->frame_id, t->alpha)) return -1;
    activated.push_back(unconfirmed[m.first]);
  }
  for (int i : u_unconf) {
    unconfirmed[i]->state = kRemoved;
    removed_new.push_back(unconfirmed[i]);
  }

  // ---- step 4: new tracks ----
  for (int i : u_det) {
    STrack& d = *dets3[i];
    if (d.score < t->det_thresh) continue;
    d.track_id = ++(*t->id_counter);               // activate :66-76 (is_activated stays False, as in the reference)
    double z[4];
    d.xyah(z);
    kf_initiate(z, d.mean, d.cov);
    d.has_mean = true;
    d.tracklet_len = 0;
    d.state = kTracked;
    d.frame_id = t->frame_id;
    d.start_frame = t->frame_id;
    activated.push_back(dets3[i]);
  }

  // ---- step 5: state update ----
  for (const TrackPtr& tr : t->lost)
    if (t->frame_id - tr->frame_id > t->max_frame_lost) {
      tr->state = kRemoved;
      removed_new.push_back(tr);
    }
  TrackList keep;
  for (const TrackPtr& tr : t->tracked)
    if (tr->state == kTracked) keep.push_back(tr);
  t->tracked = joint_stracks(joint_stracks(keep, activated), refind);
  t->lost = sub_stracks(t->lost, t->tracked);
  t->lost.insert(t->lost.end(), lost_new.begin(), lost_new.end());
  t->lost = sub_by_ids(t->lost, t->removed_ids);   // the removed list *before* this frame's removals (:343-344)
  for (const TrackPtr& tr : removed_new) t->removed_ids.insert(tr->track_id);
  {   // remove_duplicate_stracks :383-398
    iou_cost(t->tracked, t->lost, cost);
    const size_t na = t->tracked.size(), nb = t->lost.size();
    std::vector<char> dupa(na, 0), dupb(nb, 0);
    for (size_t p = 0; p < na; ++p)
      for (size_t q = 0; q < nb; ++q)
        if (cost[p * nb + q] < 0.15) {
          const int timep = t->tracked[p]->frame_id - t->tracked[p]->start_frame;
          const int timeq = t->lost[q]->frame_id - t->lost[q]->start_frame;
          if (timep > timeq) dupb[q] = 1;
          else dupa[p] = 1;
        }
    TrackList ra, rb;
    for (size_t p = 0; p < na; ++p)
      if (!dupa[p]) ra.push_back(t->tracked[p]);
    for (size_t q = 0; q < nb; ++q)
      if (!dupb[q]) rb.push_back(t->lost[q]);
    t->tracked.swap(ra);
    t->lost.swap(rb);
  }
  t->output.clear();
  for (const TrackPtr& tr : t->tracked)
    if (tr->is_activated) t->output.push_back(tr);
  return static_cast<int>(t->output.size());
}

int b2_jde_get_tracks(b2_jde* t, int which, int cap, int32_t* ids, int32_t* state, int32_t* is_activated,
                      int32_t* frame_id, int32_t* start_frame, int32_t* tracklet_len, double* tlwh, double* det_tlwh,
                      double* det_conf, double* score, double* mean, double* cov) {
  B2_CHECK(t, "b2_jde_get_tracks: null tracker");
  B2_CHECK(which >= 0 && which <= 2, "b2_jde_get_tracks: which must be 0 (output), 1 (tracked) or 2 (lost)");
  const TrackList& l = which == 0 ? t->output : which == 1 ? t->tracked : t->lost;
  const int n = static_cast<int>(l.size());
  if (cap == 0 && !ids) return n;
  B2_CHECK(cap >= n, "b2_jde_get_tracks: capacity too small");
  for (int k = 0; k < n; ++k) {
    const STrack& tr = *l[k];
    if (ids) ids[k] = tr.track_id;
    if (state) state[k] = tr.state;
    if (is_activated) is_activated[k] = tr.is_activated ? 1 : 0;
    if (frame_id) frame_id[k] = tr.frame_id;
    if (start_frame) start_frame[k] = tr.start_frame;
    if (tracklet_len) tracklet_len[k] = tr.tracklet_len;
    if (tlwh) tr.tlwh(tlwh + 4 * k);
    if (det_tlwh) memcpy(det_tlwh + 4 * k, tr.cur_det_tlwh, sizeof(double) * 4);
    if (det_conf) det_conf[k] = tr.cur_det_conf;
    if (score) score[k] = tr.score;
    if (mean) memcpy(mean + 8 * k, tr.mean, sizeof(double) * 8);
    if (cov) memcpy(cov + 64 * k, tr.cov, sizeof(double) * 64);
  }
  return n;
}

}  // extern "C"
