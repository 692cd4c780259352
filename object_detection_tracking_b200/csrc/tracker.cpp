// DeepSORT association loop in native host code (float64 state, as the reference): Kalman predict / project /
// update / gating, matching cascade, IoU matching, rectangular linear assignment, track life cycle, per-track
// appearance gallery -- with the appearance cost matrix computed on the GPU by b2_cosine_cost (one tensor-core GEMM)
// unless the caller installs another cost function.
//
// Reference (Python, per-track loops): deep_sort/tracker.py:10-138, track.py:19-166, kalman_filter.py:23-232,
// linear_assignment.py:12-194, iou_matching.py:8-81, nn_matching.py:137-177, application_util/preprocessing.py:6-74;
// scipy.optimize.linear_sum_assignment (linear_assignment.py:5,60; SciPy's rectangular shortest-augmenting-path
// solver, Crouse 2016) is restated in lsap() so that ties resolve as they do in the reference.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <deque>
#include <limits>
#include <map>
#include <memory>
#include <vector>

#include "../../include/b200det.h"
#include "common.h"

#include "assoc.h"

namespace b2 {

// ---- rectangular linear sum assignment (SciPy rectangular_lsap: shortest augmenting paths with dual variables;
// the column candidates are visited in reverse order and ties prefer an unassigned column, as SciPy does) ----
int lsap(int nr, int nc, const double* cost_in, std::vector<int>& rows, std::vector<int>& cols) {
  rows.clear();
  cols.clear();
  if (nr == 0 || nc == 0) return 0;
  const bool transpose = nc < nr;
  std::vector<double> tmp;
  const double* cost = cost_in;
  if (transpose) {
    tmp.resize(static_cast<size_t>(nr) * nc);
    for (int i = 0; i < nr; ++i)
      for (int j = 0; j < nc; ++j) tmp[static_cast<size_t>(j) * nr + i] = cost_in[static_cast<size_t>(i) * nc + j];
    cost = tmp.data();
    std::swap(nr, nc);
  }
  for (size_t i = 0; i < static_cast<size_t>(nr) * nc; ++i)
    if (cost[i] != cost[i] || cost[i] == -std::numeric_limits<double>::infinity()) return -1;
  const double inf = std::numeric_limits<double>::infinity();
  std::vector<double> u(nr, 0.0), v(nc, 0.0), spc(nc);
  std::vector<int> path(nc, -1), col4row(nr, -1), row4col(nc, -1), remaining(nc);
  std::vector<char> SR(nr), SC(nc);
  for (int cur = 0; cur < nr; ++cur) {
    double min_val = 0;
    int i = cur;
    int num_remaining = nc;
    for (int it = 0; it < nc; ++it) remaining[it] = nc - it - 1;
    std::fill(SR.begin(), SR.end(), 0);
    std::fill(SC.begin(), SC.end(), 0);
    std::fill(spc.begin(), spc.end(), inf);
    int sink = -1;
    while (sink == -1) {
      int index = -1;
      double lowest = inf;
      SR[i] = 1;
      for (int it = 0; it < num_remaining; ++it) {
        const int j = remaining[it];
        const double r = min_val + cost[static_cast<size_t>(i) * nc + j] - u[i] - v[j];
        if (r < spc[j]) {
          path[j] = i;
          spc[j] = r;
        }
        if (spc[j] < lowest || (spc[j] == lowest && row4col[j] == -1)) {
          lowest = spc[j];
          index = it;
        }
      }
      min_val = lowest;
      if (min_val == inf) return -1;   // infeasible
      const int j = remaining[index];
      if (row4col[j] == -1) sink = j;
      else i = row4col[j];
      SC[j] = 1;
      remaining[index] = remaining[--num_remaining];
    }
    u[cur] += min_val;
    for (int r = 0; r < nr; ++r)
      if (SR[r] && r != cur) u[r] += min_val - spc[col4row[r]];
    for (int j = 0; j < nc; ++j)
      if (SC[j]) v[j] -= min_val - spc[j];
    int j = sink;
    while (true) {
      const int r = path[j];
      row4col[j] = r;
      std::swap(col4row[r], j);
      if (r == cur) break;
    }
  }
  if (transpose) {   // rows of the original matrix are the columns here: report sorted by original row
    std::vector<int> order(nr);
    for (int i = 0; i < nr; ++i) order[i] = i;
    std::sort(order.begin(), order.end(), [&](int a, int b) { return col4row[a] < col4row[b]; });
    for (int k = 0; k < nr; ++k) {
      rows.push_back(col4row[order[k]]);
      cols.push_back(order[k]);
    }
  } else {
    for (int i = 0; i < nr; ++i) {
      rows.push_back(i);
      cols.push_back(col4row[i]);
    }
  }
  return 0;
}

namespace {

constexpr double kInftyCost = 1e+5;         // linear_assignment.py:9
enum { kTentative = 1, kConfirmed = 2, kDeleted = 3 };      // track.py:5-16

// ---- track state (track.py:19-166) ----
struct Track {
  double mean[8];
  double cov[64];
  int id = 0, hits = 1, age = 1, time_since_update = 0, state = kTentative;
  int n_init = 1, max_age = 60;
  std::vector<std::vector<float>> features;   // appearance vectors waiting for partial_fit (track.py:79-81)
  bool confirmed() const { return state == kConfirmed; }
  void to_tlwh(double out[4]) const {          // track.py:83-95
    out[2] = mean[2] * mean[3];
    out[3] = mean[3];
    out[0] = mean[0] - out[2] / 2;
    out[1] = mean[1] - out[3] / 2;
  }
};

struct Det {
  double tlwh[4];
  double xyah[4];
  double confidence;
  const float* feature;
};

}  // namespace
}  // namespace b2

using namespace b2;

struct b2_tracker {
  int device = 0, precision = 1;
  double max_iou_distance = 0.5, matching_threshold = 0.5;
  int max_age = 60, n_init = 1, budget = 0, feat_dim = 0;
  int next_id = 1;
  b2_appearance_cost_fn cost_fn = nullptr;
  void* cost_user = nullptr;
  std::vector<Track> tracks;
  std::map<int, std::deque<std::vector<float>>> samples;   // nn_matching.py:131 (per-target gallery)
  // scratch
  std::vector<float> gal, cost32, dfeat;
  std::vector<int32_t> seg;
};

namespace {

typedef std::vector<std::pair<int, int>> Matches;

// linear_assignment.py:12-78
int min_cost_matching(b2_tracker* t, bool appearance, double max_distance, const std::vector<Det>& dets,
                      const std::vector<int>& ti, const std::vector<int>& di, Matches& matches, std::vector<int>& ut,
                      std::vector<int>& ud) {
  matches.clear();
  ut.clear();
  ud.clear();
  if (ti.empty() || di.empty()) {
    ut = ti;
    ud = di;
    return 0;
  }
  const int T = static_cast<int>(ti.size()), N = static_cast<int>(di.size());
  std::vector<double> cost(static_cast<size_t>(T) * N);
  if (appearance) {
    // tracker.py:94-104: cosine cost of every (track gallery, detection) pair, then Mahalanobis gating
    const int D = t->feat_dim;
    t->seg.assign(T + 1, 0);
    t->gal.clear();
    for (int r = 0; r < T; ++r) {
      auto it = t->samples.find(t->tracks[ti[r]].id);
      B2_CHECK(it != t->samples.end() && !it->second.empty(), "tracker: confirmed track without a gallery");
      for (const auto& f : it->second) t->gal.insert(t->gal.end(), f.begin(), f.end());
      t->seg[r + 1] = t->seg[r] + static_cast<int32_t>(it->second.size());
    }
    t->dfeat.resize(static_cast<size_t>(N) * D);
    for (int c = 0; c < N; ++c) memcpy(&t->dfeat[static_cast<size_t>(c) * D], dets[di[c]].feature, sizeof(float) * D);
    t->cost32.resize(static_cast<size_t>(T) * N);
    int rc;
    if (t->cost_fn)
      rc = t->cost_fn(t->cost_user, t->gal.data(), t->seg.data(), T, t->dfeat.data(), N, D, t->cost32.data());
    else
      rc = b2_cosine_cost(t->device, t->gal.data(), t->seg.data(), T, t->dfeat.data(), N, D, t->precision,
                          t->cost32.data());
    if (rc != 0) return -1;
    std::vector<double> zs(static_cast<size_t>(N) * 4), g(N);
    for (int c = 0; c < N; ++c) memcpy(&zs[c * 4], dets[di[c]].xyah, sizeof(double) * 4);
    for (int r = 0; r < T; ++r) {
      const Track& tr = t->tracks[ti[r]];
      B2_CHECK(kf_gating(tr.mean, tr.cov, zs.data(), N, g.data()), "tracker: projected covariance not positive definite");
      for (int c = 0; c < N; ++c)
        cost[static_cast<size_t>(r) * N + c] = g[c] > kChi2Inv95_4 ? kInftyCost : static_cast<double>(t->cost32[static_cast<size_t>(r) * N + c]);
    }
  } else {
    // iou_matching.py:42-81
    for (int r = 0; r < T; ++r) {
      const Track& tr = t->tracks[ti[r]];
      if (tr.time_since_update > 1) {
        for (int c = 0; c < N; ++c) cost[static_cast<size_t>(r) * N + c] = kInftyCost;
        continue;
      }
      double b[4];
      tr.to_tlwh(b);
      const double area_b = b[2] * b[3];
      for (int c = 0; c < N; ++c) {
        const double* q = dets[di[c]].tlwh;
        const double tlx = std::max(b[0], q[0]), tly = std::max(b[1], q[1]);
        const double brx = std::min(b[0] + b[2], q[0] + q[2]), bry = std::min(b[1] + b[3], q[1] + q[3]);
        const double inter = std::max(0.0, brx - tlx) * std::max(0.0, bry - tly);
        cost[static_cast<size_t>(r) * N + c] = 1.0 - inter / (area_b + q[2] * q[3] - inter);
      }
    }
  }
  for (double& v : cost)
    if (v > max_distance) v = max_distance + 1e-5;
  std::vector<int> rows, cols;
  B2_CHECK(lsap(T, N, cost.data(), rows, cols) == 0, "tracker: linear assignment failed (non-finite cost)");
  std::vector<char> row_used(T, 0), col_used(N, 0);
  for (size_t k = 0; k < rows.size(); ++k) {
    row_used[rows[k]] = 1;
    col_used[cols[k]] = 1;
  }
  for (int c = 0; c < N; ++c)
    if (!col_used[c]) ud.push_back(di[c]);
  for (int r = 0; r < T; ++r)
    if (!row_used[r]) ut.push_back(ti[r]);
  for (size_t k = 0; k < rows.size(); ++k) {
    if (cost[static_cast<size_t>(rows[k]) * N + cols[k]] > max_distance) {
      ut.push_back(ti[rows[k]]);
      ud.push_back(di[cols[k]]);
    } else {
      matches.push_back(std::make_pair(ti[rows[k]], di[cols[k]]));
    }
  }
  return 0;
}

}  // namespace

extern "C" {

int b2_tracker_create(b2_tracker** out, int device, double max_iou_distance, int max_age, int n_init,
                      double matching_threshold, int budget, int feat_dim, int precision) {
  B2_CHECK(out, "b2_tracker_create: null argument");
  *out = nullptr;
  B2_CHECK(feat_dim > 0 && max_age >= 0 && n_init >= 0, "b2_tracker_create: bad parameters");
  b2_tracker* t = new b2_tracker();
  t->device = device;
  t->precision = precision;
  t->max_iou_distance = max_iou_distance;
  t->max_age = max_age;
  t->n_init = n_init;
  t->matching_threshold = matching_threshold;
  t->budget = budget;
  t->feat_dim = feat_dim;
  *out = t;
  return 0;
}

void b2_tracker_destroy(b2_tracker* t) { delete t; }

int b2_tracker_set_cost_fn(b2_tracker* t, b2_appearance_cost_fn fn, void* user) {
  B2_CHECK(t, "b2_tracker_set_cost_fn: null tracker");
  t->cost_fn = fn;
  t->cost_user = user;
  return 0;
}

int b2_tracker_predict(b2_tracker* t) {   // tracker.py:50-56, track.py:107-124
  B2_CHECK(t, "b2_tracker_predict: null tracker");
  for (Track& tr : t->tracks) {
    kf_predict(tr.mean, tr.cov);
    tr.age += 1;
    tr.time_since_update += 1;
  }
  return 0;
}

int b2_tracker_update(b2_tracker* t, const double* tlwh, const double* confidence, const float* features, int n) {
  B2_CHECK(t && (n == 0 || (tlwh && features)), "b2_tracker_update: null argument");
  const int D = t->feat_dim;
  std::vector<Det> dets(n);
  for (int i = 0; i < n; ++i) {
    Det& d = dets[i];
    memcpy(d.tlwh, tlwh + 4 * i, sizeof(double) * 4);
    d.xyah[0] = d.tlwh[0] + d.tlwh[2] / 2;        // detection.py:44-49
    d.xyah[1] = d.tlwh[1] + d.tlwh[3] / 2;
    d.xyah[2] = d.tlwh[2] / d.tlwh[3];
    d.xyah[3] = d.tlwh[3];
    d.confidence = confidence ? confidence[i] : 1.0;
    d.feature = features + static_cast<size_t>(i) * D;
  }
  // ---- tracker.py:92-131 _match ----
  std::vector<int> confirmed, unconfirmed;
  for (int k = 0; k < static_cast<int>(t->tracks.size()); ++k)
    (t->tracks[k].confirmed() ? confirmed : unconfirmed).push_back(k);
  // matching cascade (linear_assignment.py:81-145)
  std::vector<int> ud(n);
  for (int i = 0; i < n; ++i) ud[i] = i;
  Matches matches_a, m;
  std::vector<int> ut_tmp, ud_tmp;
  for (int level = 0; level < t->max_age; ++level) {
    if (ud.empty()) break;
    std::vector<int> lvl;
    for (int k : confirmed)
      if (t->tracks[k].time_since_update == 1 + level) lvl.push_back(k);
    if (lvl.empty()) continue;
    if (min_cost_matching(t, true, t->matching_threshold, dets, lvl, ud, m, ut_tmp, ud_tmp)) return -1;
    matches_a.insert(matches_a.end(), m.begin(), m.end());
    ud = ud_tmp;
  }
  std::vector<char> matched(t->tracks.size(), 0);
  for (const auto& pr : matches_a) matched[pr.first] = 1;
  std::vector<int> iou_cand = unconfirmed, ut_a;
  for (int k : confirmed) {
    if (matched[k]) continue;
    if (t->tracks[k].time_since_update == 1) iou_cand.push_back(k);
    else ut_a.push_back(k);
  }
  Matches matches_b;
  std::vector<int> ut_b;
  if (min_cost_matching(t, false, t->max_iou_distance, dets, iou_cand, ud, matches_b, ut_b, ud_tmp)) return -1;
  ud = ud_tmp;
  Matches matches = matches_a;
  matches.insert(matches.end(), matches_b.begin(), matches_b.end());
  std::vector<int> ut = ut_a;
  ut.insert(ut.end(), ut_b.begin(), ut_b.end());
  // ---- tracker.py:57-90 update ----
  for (const auto& pr : matches) {             // track.py:126-145
    Track& tr = t->tracks[pr.first];
    const Det& d = dets[pr.second];
    B2_CHECK(kf_update(tr.mean, tr.cov, d.xyah), "tracker: innovation covariance not positive definite");
    tr.features.emplace_back(d.feature, d.feature + D);
    tr.hits += 1;
    tr.time_since_update = 0;
    if (tr.state == kTentative && tr.hits >= tr.n_init) tr.state = kConfirmed;
  }
  for (int k : ut) {                           // track.py:147-153
    Track& tr = t->tracks[k];
    if (tr.state == kTentative || tr.time_since_update > tr.max_age) tr.state = kDeleted;
  }
  for (int di : ud) {                          // tracker.py:133-138
    Track tr;
    kf_initiate(dets[di].xyah, tr.mean, tr.cov);
    tr.id = t->next_id++;
    tr.n_init = t->n_init;
    tr.max_age = t->max_age;
    tr.features.emplace_back(dets[di].feature, dets[di].feature + D);
    t->tracks.push_back(std::move(tr));
  }
  t->tracks.erase(std::remove_if(t->tracks.begin(), t->tracks.end(), [](const Track& tr) { return tr.state == kDeleted; }),
                  t->tracks.end());
  // distance metric bookkeeping (tracker.py:79-90, nn_matching.py:137-154)
  std::map<int, std::deque<std::vector<float>>> next;
  for (Track& tr : t->tracks) {
    if (!tr.confirmed()) continue;
    auto it = t->samples.find(tr.id);
    std::deque<std::vector<float>>& g = next[tr.id];
    if (it != t->samples.end()) g.swap(it->second);
    for (auto& f : tr.features) {
      g.push_back(std::move(f));
      if (t->budget > 0)
        while (static_cast<int>(g.size()) > t->budget) g.pop_front();
    }
    tr.features.clear();
  }
  t->samples.swap(next);
  return 0;
}

int b2_tracker_num_tracks(b2_tracker* t) { return t ? static_cast<int>(t->tracks.size()) : -1; }

int b2_tracker_get_tracks(b2_tracker* t, int cap, int32_t* ids, int32_t* state, int32_t* hits, int32_t* age,
                          int32_t* time_since_update, double* mean, double* cov) {
  B2_CHECK(t, "b2_tracker_get_tracks: null tracker");
  const int n = static_cast<int>(t->tracks.size());
  B2_CHECK(cap >= n, "b2_tracker_get_tracks: capacity too small");
  for (int k = 0; k < n; ++k) {
    const Track& tr = t->tracks[k];
    if (ids) ids[k] = tr.id;
    if (state) state[k] = tr.state;
    if (hits) hits[k] = tr.hits;
    if (age) age[k] = tr.age;
    if (time_since_update) time_since_update[k] = tr.time_since_update;
    if (mean) memcpy(mean + 8 * k, tr.mean, sizeof(double) * 8);
    if (cov) memcpy(cov + 64 * k, tr.cov, sizeof(double) * 64);
  }
  return n;
}

int b2_linear_sum_assignment(const double* cost, int nr, int nc, int32_t* rows, int32_t* cols) {
  B2_CHECK(nr >= 0 && nc >= 0 && (nr == 0 || nc == 0 || cost), "b2_linear_sum_assignment: bad argument");
  std::vector<int> r, c;
  B2_CHECK(lsap(nr, nc, cost, r, c) == 0, "b2_linear_sum_assignment: infeasible or non-finite cost matrix");
  for (size_t k = 0; k < r.size(); ++k) {
    rows[k] = r[k];
    cols[k] = c[k];
  }
  return static_cast<int>(r.size());
}

// application_util/preprocessing.py:6-74 (pre-tracker NMS): greedy by ascending score order from the back, overlap
// = intersection / area of the *other* box with the +1 pixel convention.
int b2_track_nms(const double* tlwh, const double* scores, int n, double max_bbox_overlap, int32_t* keep) {
  B2_CHECK(n == 0 || (tlwh && keep), "b2_track_nms: null argument");
  std::vector<double> x1(n), y1(n), x2(n), y2(n), area(n);
  for (int i = 0; i < n; ++i) {
    x1[i] = tlwh[4 * i];
    y1[i] = tlwh[4 * i + 1];
    x2[i] = tlwh[4 * i + 2] + tlwh[4 * i];
    y2[i] = tlwh[4 * i + 3] + tlwh[4 * i + 1];
    area[i] = (x2[i] - x1[i] + 1) * (y2[i] - y1[i] + 1);
  }
  std::vector<int> idxs(n);
  for (int i = 0; i < n; ++i) idxs[i] = i;
  const double* key = scores ? scores : y2.data();
  std::stable_sort(idxs.begin(), idxs.end(), [&](int a, int b) { return key[a] < key[b]; });
  int nk = 0;
  while (!idxs.empty()) {
    const int i = idxs.back();
    idxs.pop_back();
    keep[nk++] = i;
    std::vector<int> rest;
    for (int j : idxs) {
      const double w = std::max(0.0, std::min(x2[i], x2[j]) - std::max(x1[i], x1[j]) + 1);
      const double h = std::max(0.0, std::min(y2[i], y2[j]) - std::max(y1[i], y1[j]) + 1);
      if (!((w * h) / area[j] > max_bbox_overlap)) rest.push_back(j);
    }
    idxs.swap(rest);
  }
  return nk;
}

}  // extern "C"
