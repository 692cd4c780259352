// libb200det detector engine: context, weight packing, the static per-frame launch plan, C ABI.
//
// The plan is built once per (batch, H, W): every activation buffer, every TMA tensor map and every
// kernel parameter block is fixed, so one frame is a fixed sequence of ~150 launches that is captured
// into a CUDA graph and replayed.  Graph structure follows Mask_RCNN_FPN.build_forward
// (models.py:488-973); citations at each phase.
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "../../include/b200det.h"
#include "detplan.h"
#include "planes.cuh"
#include "tf_resize_math.h"

namespace b2 {
namespace {

__global__ void subsample2_kernel(const __half* __restrict__ in_hi, const __half* __restrict__ in_lo, int B, int H,
                                  int W, int C, __half* __restrict__ out_hi, __half* __restrict__ out_lo, int Ho,
                                  int Wo) {
  const int cvec = C / 8;
  const size_t total = static_cast<size_t>(B) * Ho * Wo * cvec;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(idx % cvec);
    const size_t pix = idx / cvec;
    const int b = static_cast<int>(pix / (static_cast<size_t>(Ho) * Wo));
    const int rem = static_cast<int>(pix % (static_cast<size_t>(Ho) * Wo));
    const int p = rem / Wo, q = rem % Wo;
    const size_t src = ((static_cast<size_t>(b) * H + 2 * p) * W + 2 * q) * C + cv * 8;
    *reinterpret_cast<uint4*>(out_hi + pix * C + cv * 8) = *reinterpret_cast<const uint4*>(in_hi + src);
    if (out_lo) *reinterpret_cast<uint4*>(out_lo + pix * C + cv * 8) = *reinterpret_cast<const uint4*>(in_lo + src);
  }
}

// mean over the 7x7 bins of fpn_box_feat (deep_sort/utils.py:27-28 does this on the host)
__global__ void pool_feat_kernel(const float* __restrict__ feat, int rows, int C, float* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * C) return;
  const float* f = feat + static_cast<size_t>(idx) * 49;
  float s = 0.f;
  for (int i = 0; i < 49; ++i) s += f[i];
  out[idx] = s / 49.f;
}

// The TMOT driver's other embedding aggregations of fpn_box_feat (obj_detect_tracking_multi_queuer_tmot.py:511-525):
// mode 2 "max" = amax over the 7x7 bins -> [rows][C]; mode 3 "spatial" = mean over the channels -> [rows][49].
__global__ void agg_feat_kernel(const float* __restrict__ feat, int rows, int C, int mode, float* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (mode == 2) {
    if (idx >= rows * C) return;
    const float* f = feat + static_cast<size_t>(idx) * 49;
    float m = f[0];
    for (int i = 1; i < 49; ++i) m = fmaxf(m, f[i]);
    out[idx] = m;
  } else {
    if (idx >= rows * 49) return;
    const int r = idx / 49, bin = idx - r * 49;
    const float* f = feat + static_cast<size_t>(r) * C * 49 + bin;
    float s = 0.f;
    for (int ch = 0; ch < C; ++ch) s += f[static_cast<size_t>(ch) * 49];
    out[idx] = s / static_cast<float>(C);
  }
}

// The scene feature fpn_feature (models.py:517-518): p5 resized to 7 x 7 with TF1's legacy bilinear (tf_resize_math.h),
// float32 NHWC [B][7][7][C].  Samples the p5 of the padded image, ph x pw, out of planes of pitch pitch_h x pitch_w; below
// 7 px the resize upsamples and the clamp of the upper tap to ph - 1 / pw - 1 applies.  One thread = 8 channels of one
// output pixel.
__global__ void fpn_feature_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo, int B, int pitch_h,
                                   int pitch_w, int C, int ph, int pw, float sy, float sx, float* __restrict__ out) {
  const int cvec = C / 8;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * 49 * cvec) return;
  const int cv = idx % cvec, pix = idx / cvec;   // pix = (b * 7 + oy) * 7 + ox
  const int ox = pix % 7, oy = (pix / 7) % 7, b = pix / 49;
  const TfResizeTap ty = tf_resize_tap(oy, sy, ph), tx = tf_resize_tap(ox, sx, pw);
  const size_t img = static_cast<size_t>(b) * pitch_h * pitch_w;
  auto at = [&](int y, int x) { return (img + static_cast<size_t>(y) * pitch_w + x) * C + cv * 8; };
  float tl[8], tr[8], bl[8], br[8], r[8];
  load8(hi, lo, at(ty.lo, tx.lo), tl);
  load8(hi, lo, at(ty.lo, tx.hi), tr);
  load8(hi, lo, at(ty.hi, tx.lo), bl);
  load8(hi, lo, at(ty.hi, tx.hi), br);
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = tf_resize_lerp(tl[j], tr[j], bl[j], br[j], tx.lerp, ty.lerp);
  float4* o = reinterpret_cast<float4*>(out + static_cast<size_t>(pix) * C + cv * 8);
  o[0] = make_float4(r[0], r[1], r[2], r[3]);
  o[1] = make_float4(r[4], r[5], r[6], r[7]);
}

// The use_cpu_nms outputs of one image (models.py:899-912): the decoded, clipped boxes [K][nc1][4] transposed to
// [nc1][n][4] and the probabilities' class columns [K][1 + nc1] to [nc1][n], n = *count proposals.
__global__ void all_boxes_kernel(const float4* __restrict__ dec, const float* __restrict__ probs,
                                 const int* __restrict__ count, int K, int nc1, int ncls, float4* __restrict__ out_boxes,
                                 float* __restrict__ out_probs) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nc1 * K) return;
  const int n = *count, c = idx / K, k = idx - c * K;
  if (k >= n) return;
  out_boxes[static_cast<size_t>(c) * n + k] = dec[static_cast<size_t>(k) * nc1 + c];
  out_probs[static_cast<size_t>(c) * n + k] = probs[static_cast<size_t>(k) * ncls + c + 1];
}

enum { NPHASE = 8 };

}  // namespace
}  // namespace b2

using namespace b2;

struct b2_ctx {
  DetPlan plan;            // first member: its arena is freed after everything that refers to it
  b2_config cfg;
  b2_config_ext ext;       // options appended after b2_config's layout was fixed (b2_create_ex)
  b2_config_ext2 ext2;     // and after b2_config_ext's (b2_create_ex2)
  b2_config_ext3 ext3;     // and after b2_config_ext2's (b2_create_ex3)
  b2_config_ext4 ext4;     // and after b2_config_ext3's (b2_create_ex4)
  b2_config_ext5 ext5;     // and after b2_config_ext4's (b2_create_ex5)
  int device = 0, num_sms = 132;
  cudaStream_t stream = nullptr;
  // geometry
  int c1h = 0, c1w = 0, ch[4], cw[4], ph[5], pw[5], pfh[5], pfw[5];
  // buffers
  void* img = nullptr;
  size_t img_bytes = 0;
  uint8_t* raw_frames = nullptr;   // b2_detect_host_resize: source-resolution uint8 frames
  size_t raw_bytes = 0;
  // pipelined ingest (b2_submit_host / b2_wait): two staging buffers fed by a copy stream
  cudaStream_t copy_stream = nullptr, down_stream = nullptr;
  void* stage_in[2] = {nullptr, nullptr};
  uint8_t* stage_out[2] = {nullptr, nullptr};     // boxes | probs | labels | count | feat, device copies per slot
  cudaEvent_t pass_done[2] = {nullptr, nullptr};
  cudaEvent_t h2d_done[2] = {nullptr, nullptr}, staged_free[2] = {nullptr, nullptr}, out_done[2] = {nullptr, nullptr};
  bool slot_busy[2] = {false, false};
  // range monitor: conv_tc_kernel ORs the device word plan.range_flag when an fp16-plane output exceeds +-65504 (or is
  // NaN); the word is read back with every host-facing result (h_range: [0], [1] = submit slots, [2] = synchronous calls)
  unsigned int* h_range = nullptr;
  Planes stem_u, c1, pool, cfeat[4], lat[4], pfeat[5], rpn_h[5];
  float* rpn_out[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  RpnParams rpn;
  RoiAlignParams roi1, roi2;
  HeadPostParams post;
  Planes roi_feat, fc6, fc7;        // fc6 / fc7: the M = B * rpn_topk head rows (DetPlan::alloc_rows)
  Planes head_a, head_b;           // conv box head (cfg.conv_head_dim > 0): [M][7][7][conv_head_dim] ping-pong
  Planes rm1, rm2;                 // relation modules (cfg.add_relation_nn): their sums
  Planes att_pool, att, att_sum;   // attention head (ext3.use_att_frcnn_head): bin sums [M][256], relu(att_trans), the sum
  // small-object branch (ext4.use_small_object_head): its parameters, rows and final selection
  SoParams so;
  HeadPostParams so_fin;
  Planes so_roi, so_fc6, so_fc7, so_asso;
  float* head_logits = nullptr;
  float* box_feat = nullptr;
  float* box_feat_pooled = nullptr;
  float* given_boxes = nullptr;    // b2_box_features: [R][4] boxes + count of the current chunk
  int* given_count = nullptr;
  float* given_feat = nullptr;     // [R][C][7][7] and pooled [R][C]
  float* given_pooled = nullptr;
  float* box_feat_agg = nullptr;   // feat_mode 2 / 3 scratch ([B*R][C] or [B*R][49]), allocated on first use
  // mask head (cfg.add_mask): ROIAlign 14 of the final boxes -> 4 x conv3x3 -> deconv -> conv1x1 -> sigmoid of own class
  Planes mask_a, mask_b, mask_up;
  float* mask_logits = nullptr;
  int mask_ld = 0;
  float* final_masks = nullptr;    // [B][R][28][28]
  cudaGraphExec_t graph = nullptr;
  // b2_fpn_feature: the resized p5 [B][7][7][C], and the graph of the backbone-only pass
  float* fpn_feat = nullptr;
  cudaGraphExec_t feat_graph = nullptr;
  // b2_get_all_boxes: one image's re-laid-out boxes [nc1][K][4] and probabilities [nc1][K], allocated on first use
  float* all_boxes = nullptr;
  float* all_probs = nullptr;
  // dual-stream pass (plan.dual): the backbone / FPN / RPN-head phases run as plan.nsplit batch parts on as many streams,
  // so that the tail of one layer's persistent kernel (tiles % SMs != 0, no SM busy in the last round) overlaps the other
  // parts' kernels
  cudaStream_t side_stream[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t fork_ev = nullptr, join_ev[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  bool weights_loaded = false;
  cudaEvent_t ev[NPHASE + 1];
  float phase_ms[NPHASE];
};

namespace {

// generate_anchors.py:42-109 restated for one (stride, size): the 3 ratio anchors of a cell.
void cell_anchors(float stride, float size, const float* ratios, float out[3][4]) {
  const double base = stride;
  const double w0 = base, h0 = base, xc = 0.5 * (w0 - 1), yc = 0.5 * (h0 - 1);
  const double area = w0 * h0;
  const double scale = size / stride;
  for (int i = 0; i < 3; ++i) {
    const double ws = nearbyint(sqrt(area / ratios[i]));
    const double hs = nearbyint(ws * ratios[i]);
    // _mkanchors then _scale_enum (single scale)
    const double x1 = xc - 0.5 * (ws - 1), x2 = xc + 0.5 * (ws - 1);
    const double y1 = yc - 0.5 * (hs - 1), y2 = yc + 0.5 * (hs - 1);
    const double w = x2 - x1 + 1, h = y2 - y1 + 1;
    const double cx = x1 + 0.5 * (w - 1), cy = y1 + 0.5 * (h - 1);
    const double W = w * scale, H = h * scale;
    out[i][0] = static_cast<float>(cx - 0.5 * (W - 1));
    out[i][1] = static_cast<float>(cy - 0.5 * (H - 1));
    out[i][2] = static_cast<float>(cx + 0.5 * (W - 1));
    out[i][3] = static_cast<float>(cy + 0.5 * (H - 1));
  }
}

// The small-object branch (models.py:590-692, 845-897), phase 6 after the head's post-processing.  Rows: C blocks of
// R = result_per_im rows (small class i's NMS selections, in selection order), then Tp = so_person_topk person rows with
// use_so_association.  Steps:
//   so_select     the C (+ Person) class columns of the head: probabilities and unclipped decoded boxes; per-class NMS
//                 without a score threshold, at most R per small class and Tp for Person (head.cu's class_nms_kernel)
//   so_gather     the rows' boxes; K = the small classes' common count, or 0 with status 1 when they differ
//   so_roialign   ROIAlign 7 of the rows (unclipped boxes: samples outside the level read 0, as crop_and_resize)
//   fc6, fc7      the head's own layers (same packed weights) over all rows
//   association   person_object_relation of the C * R rows against the person rows (add_so_association)
//   classification one N = 2C fp32 layer over the C * R rows; row block i keeps its columns 2i, 2i + 1
//   so_finish     the [K][C + 1] logits and clipped [K][C][4] boxes, then the head's per-class NMS and top-k over them,
//                 with the score threshold only with use_so_score_thres: the scores are logits, not probabilities
int add_small_objects(b2_ctx* c, const ConvLayer* fc6, const ConvLayer* fc7) {
  const b2_config& cfg = c->cfg;
  const b2_config_ext4& e = c->ext4;
  DetPlan& P = c->plan;
  B2_CHECK(fc6 && fc7, "b2_create: use_small_object_head needs the 2fc box head");
  const int C = e.num_small_objects, R = cfg.result_per_im, K = cfg.rpn_topk, nc = cfg.fpn_num_channel;
  const int Tp = e.use_so_association ? e.so_person_topk : 0, SR = C * R + Tp, dim = cfg.fc_head_dim;
  const HeadPostParams& hp = c->post;
  SoParams& sp = c->so;
  memset(&sp, 0, sizeof(sp));
  sp.logits = hp.logits; sp.ld = hp.ld; sp.num_class = hp.num_class; sp.rois = K;
  sp.roi_boxes = hp.rois; sp.roi_count = hp.roi_count; sp.probs = hp.probs;
  for (int i = 0; i < 4; ++i) sp.reg_w[i] = hp.reg_w[i];
  sp.decode_clip = hp.decode_clip; sp.img_w = hp.img_w; sp.img_h = hp.img_h;
  sp.C = C; sp.R = R; sp.Tp = Tp;
  for (int i = 0; i < C; ++i) sp.ids[i] = e.small_object_class_ids[i];
  if (Tp) sp.ids[C] = e.so_person_class_id;
  sp.sel_probs = P.arena.alloc<float>(static_cast<size_t>(K) * (C + 2));
  sp.sel_boxes = P.arena.alloc<float>(static_cast<size_t>(K) * (C + 1) * 4);
  int* keep = P.arena.alloc<int>(static_cast<size_t>(C + 1) * R);
  int* pkeep = P.arena.alloc<int>(static_cast<size_t>(C + 1) * std::max(Tp, 1));
  int* sel_count = P.arena.alloc<int>(C + 1);
  sp.keep = keep; sp.person_keep = pkeep + static_cast<size_t>(C) * Tp; sp.sel_count = sel_count;
  sp.rows_boxes = P.arena.alloc<float>(static_cast<size_t>(SR) * 4);
  sp.row_count = P.arena.alloc<int>(C + 1);
  sp.k = P.arena.alloc<int>(1);
  sp.status = P.arena.alloc<int>(1);
  B2_CHECK(sp.sel_probs && sp.sel_boxes && keep && pkeep && sel_count && sp.rows_boxes && sp.row_count && sp.k && sp.status,
           "out of device memory (small-object selection)");
  // the selection's NMS: head.cu's kernel over the gathered columns, class s at dec_boxes column s, probs column s + 1
  HeadPostParams sel = hp;
  sel.probs = sp.sel_probs; sel.dec_boxes = sp.sel_boxes; sel.num_class = C + 2;
  sel.score_thresh = -INFINITY;   // nms_return_boxes / the person NMS have no score threshold (models.py:1240-1250, 654-656)
  sel.max_per_class = R; sel.cls_keep = keep; sel.cls_count = sel_count;
  sel.bg_rank = nullptr;          // nms_return_boxes has no background filter (models.py:1240-1250)
  HeadPostParams psel = sel;
  psel.max_per_class = std::max(Tp, 1); psel.cls_keep = pkeep;
  Step& s1 = add_batch_step(P, 6, kStepSoSelect, "", [c, sel, psel](int, int, cudaStream_t st) {
    if (so_select_launch(c->so, st) || class_nms_launch(sel, 0, c->so.C, st)) return -1;
    return c->so.Tp ? class_nms_launch(psel, c->so.C, 1, st) : 0;
  }, Tp ? 3 : 2);
  s1.bytes = static_cast<double>(K) * (hp.ld + 2.0 * (C + 2) + 8.0 * (C + 1)) * 4;
  add_batch_step(P, 6, kStepSoGather, "", [c](int, int, cudaStream_t st) { return so_gather_launch(c->so, st); });
  // ROIAlign of the rows: the C class blocks as C groups of R rows (of the one image), then the Tp person rows
  B2_CHECK(P.alloc_rows(c->so_roi, SR, 49 * nc) && P.alloc_rows(c->so_fc6, SR, dim) && P.alloc_rows(c->so_fc7, SR, dim),
           "alloc small-object rows");
  RoiAlignParams ra = c->roi1;
  ra.B = C; ra.rois_per_image = R; ra.one_image = 1;
  ra.boxes = sp.rows_boxes; ra.count = sp.row_count;
  ra.out_hi = c->so_roi.hi; ra.out_lo = c->so_roi.lo;
  RoiAlignParams rb = ra;
  const size_t off = static_cast<size_t>(C) * R * 49 * nc;
  rb.B = 1; rb.rois_per_image = Tp;
  rb.boxes = sp.rows_boxes + static_cast<size_t>(C) * R * 4; rb.count = sp.row_count + C;
  rb.out_hi = c->so_roi.hi + off; rb.out_lo = c->so_roi.lo ? c->so_roi.lo + off : nullptr;
  add_batch_step(P, 6, kStepSoRoialign, "", [ra, rb](int, int, cudaStream_t st) {
    if (roialign_launch(ra, st)) return -1;
    return rb.rois_per_image > 0 ? roialign_launch(rb, st) : 0;
  }, Tp ? 2 : 1).bytes = static_cast<double>(SR) * 49 * nc * (P.split ? 4.0 : 2.0) * 2;
  if (!add_conv_shared(P, 6, "fastrcnn/small_objects/fc6", c->so_roi, *fc6, c->so_fc6) ||
      !add_conv_shared(P, 6, "fastrcnn/small_objects/fc7", c->so_fc6, *fc7, c->so_fc7))
    return -1;
  Planes hidden = c->so_fc7;
  hidden.W = C * R;
  if (Tp) {
    B2_CHECK(P.alloc_rows(c->so_asso, C * R, dim), "alloc small-object association rows");
    if (add_so_association(P, 6, "fastrcnn/small_objects/person_object_relation", C, R, Tp, sp.rows_boxes, sp.k,
                           sp.row_count + C, c->so_fc7, c->so_asso))
      return -1;
    hidden = c->so_asso;
  }
  sp.ldl = (2 * C + 15) / 16 * 16;
  float* cls = P.arena.alloc<float>(static_cast<size_t>((C * R + 127) / 128 * 128) * sp.ldl);
  sp.fin_logits = P.arena.alloc<float>(static_cast<size_t>(R) * (C + 1));
  sp.fin_boxes = P.arena.alloc<float>(static_cast<size_t>(R) * C * 4);
  sp.cls_logits = cls;
  add_conv_f32(P, 6, "fastrcnn/small_objects/classification", hidden, conv_desc(1, 2 * C), kBias, cls, sp.ldl, kSoClass);
  HeadPostParams& fin = c->so_fin;
  memset(&fin, 0, sizeof(fin));
  fin.probs = sp.fin_logits; fin.dec_boxes = sp.fin_boxes; fin.num_class = C + 1; fin.B = 1; fin.rois_per_image = R;
  fin.roi_count = sp.k;
  fin.score_thresh = e.use_so_score_thres ? cfg.result_score_thres : -INFINITY;   // models.py:880-884
  fin.nms_thr = cfg.fastrcnn_nms_iou_thres;
  fin.max_per_class = R; fin.max_total = R;
  fin.cls_keep = P.arena.alloc<int>(static_cast<size_t>(C) * R);
  fin.cls_count = P.arena.alloc<int>(C);
  fin.final_boxes = P.arena.alloc<float>(static_cast<size_t>(R) * 4);
  fin.final_probs = P.arena.alloc<float>(R);
  fin.final_labels = P.arena.alloc<int>(R);
  fin.final_count = P.arena.alloc<int>(1);
  B2_CHECK(cls && sp.fin_logits && sp.fin_boxes && fin.cls_keep && fin.cls_count && fin.final_boxes && fin.final_probs &&
               fin.final_labels && fin.final_count, "out of device memory (small-object outputs)");
  // use_bg_score: the branch's fastrcnn_predictions filters too, on the argmax of the rebuilt logits (models.py:885-889)
  if (c->post.bg_rank) {
    fin.bg_rank = P.arena.alloc<int>(R);
    B2_CHECK(fin.bg_rank, "out of device memory (small-object background filter)");
    P.stages.raw("so_bg_rank", fin.bg_rank, Stage::kI32, R, 1, 1, 1);
  }
  add_batch_step(P, 6, kStepSoFinish, "", [c](int, int, cudaStream_t st) {
    if (so_finish_launch(c->so, st)) return -1;
    return head_select_launch(c->so_fin, st);
  }, fin.bg_rank ? 4 : 3);
  P.stages.raw("so_sel_probs", sp.sel_probs, Stage::kF32, K, C + 2, 1, 1);
  P.stages.raw("so_sel_boxes", sp.sel_boxes, Stage::kF32, K, C + 1, 4, 1);
  P.stages.raw("so_sel_count", sel_count, Stage::kI32, C + 1, 1, 1, 1);
  P.stages.raw("so_keep", keep, Stage::kI32, C, R, 1, 1);
  P.stages.raw("so_person_keep", pkeep + static_cast<size_t>(C) * Tp, Stage::kI32, std::max(Tp, 1), 1, 1, 1);
  P.stages.raw("so_status", sp.status, Stage::kI32, 1, 1, 1, 1);
  P.stages.raw("so_k", sp.k, Stage::kI32, 1, 1, 1, 1);
  P.stages.raw("so_boxes", sp.rows_boxes, Stage::kF32, SR, 4, 1, 1);
  P.stages.planes("so_roi_feat", c->so_roi);
  P.stages.planes("so_fc6", c->so_fc6);
  P.stages.planes("so_fc7", c->so_fc7);
  if (Tp) P.stages.planes("so_asso", c->so_asso);
  P.stages.raw("so_cls_logits", cls, Stage::kF32, C * R, sp.ldl, 1, 1);
  P.stages.raw("so_logits", sp.fin_logits, Stage::kF32, R, C + 1, 1, 1);
  P.stages.raw("so_final_boxes", fin.final_boxes, Stage::kF32, R, 4, 1, 1);
  P.stages.raw("so_final_probs", fin.final_probs, Stage::kF32, R, 1, 1, 1);
  P.stages.raw("so_final_labels", fin.final_labels, Stage::kI32, R, 1, 1, 1);
  P.stages.raw("so_final_count", fin.final_count, Stage::kI32, 1, 1, 1, 1);
  return 0;
}

int build_plan(b2_ctx* c) {
  const b2_config& cfg = c->cfg;
  const int B = cfg.batch, H = cfg.height, W = cfg.width;
  B2_CHECK(B >= 1 && H >= 32 && W >= 32, "b2_create: bad frame geometry");
  B2_CHECK(cfg.fpn_num_channel == 256, "b2_create: fpn_num_channel must be 256");
  B2_CHECK(cfg.rpn_topk >= 1 && cfg.rpn_topk <= 1024, "b2_create: rpn_topk must be in [1,1024]");
  DetPlan& P = c->plan;
  P.batch = B;
  P.conv_impl = cfg.conv_impl;
  P.acc_kb = cfg.accum_chunk;
  // Images are independent through phases 0-2 (stem, ResNet, FPN, RPN head): their steps also get one launch per part of
  // the batch, each with its own plans (same tiles per image, so the results are bit-identical to the full-batch plan).
  if (cfg.conv_impl == 0) {
    P.nsplit = 2;
    if (const char* e = getenv("B2_SPLIT")) P.nsplit = atoi(e);   // experiment hook: 1, 2, 4, 8 batch parts
    if (P.nsplit < 1 || P.nsplit > 8 || B % P.nsplit != 0) P.nsplit = 1;
    P.dual = P.nsplit > 1;
  }
  // ---- geometry (nn.py:843-944, tf_pad_reverse=True) ----
  const int PH = (H + 31) / 32 * 32, PW = (W + 31) / 32 * 32;
  c->c1h = (PH + 5 - 7) / 2 + 1;
  c->c1w = (PW + 5 - 7) / 2 + 1;
  int h = (c->c1h + 1 - 3) / 2 + 1, w = (c->c1w + 1 - 3) / 2 + 1;
  for (int g = 0; g < 4; ++g) {
    if (g > 0) { h = (h + 1 - 3) / 2 + 1; w = (w + 1 - 3) / 2 + 1; }
    c->ch[g] = h; c->cw[g] = w;
  }
  for (int i = 0; i < 4; ++i) { c->pfh[i] = c->ch[i]; c->pfw[i] = c->cw[i]; }
  c->pfh[4] = (c->ch[3] - 1) / 2 + 1;
  c->pfw[4] = (c->cw[3] - 1) / 2 + 1;
  for (int i = 0; i < 5; ++i) {
    c->ph[i] = c->pfh[i]; c->pw[i] = c->pfw[i];
    if (i < 3) {   // models.py:382-390 crop p2..p4 to ceil(H/stride)
      const int s = static_cast<int>(cfg.anchor_strides[i]);
      c->ph[i] = std::min(c->pfh[i], (H + s - 1) / s);
      c->pw[i] = std::min(c->pfw[i], (W + s - 1) / s);
    }
  }
  for (int i = 0; i < 3; ++i)
    B2_CHECK(c->ch[i] == 2 * c->ch[i + 1] && c->cw[i] == 2 * c->cw[i + 1], "b2_create: FPN levels must nest 2x");

  // ---- input + stem + pool (phase 0) ----
  c->img_bytes = static_cast<size_t>(B) * H * W * 3 * (cfg.input_dtype == 1 ? 1 : 4);
  c->img = P.arena.alloc<uint8_t>(c->img_bytes);
  P.range_flag = P.arena.alloc<unsigned int>(1);
  B2_CHECK(P.range_flag != nullptr, "out of device memory (range flag)");
  B2_CUDA(cudaMallocHost(&c->h_range, 3 * sizeof(unsigned int)));
  c->h_range[0] = c->h_range[1] = c->h_range[2] = 0;
  // compact stem operand [B][c1h + 3][c1w + 3][16]; conv0 reads 64-channel pixels out of it with a pixel stride of 16 (stem.cu)
  B2_CHECK(P.alloc_planes(c->stem_u, B, c->c1h + 3, c->c1w + 3, 16), "alloc stem operand");
  B2_CHECK(P.alloc_planes(c->c1, B, c->c1h, c->c1w, 64), "alloc c1");
  B2_CHECK(P.alloc_planes(c->pool, B, c->ch[0], c->cw[0], 64), "alloc pool");
  const double esz = P.split ? 4.0 : 2.0;
  add_batch_step(P, 0, kStepStemPack, "", [c](int b0, int n, cudaStream_t st) {
    const Planes u = c->stem_u.images(b0, n);
    return stem_pack16_launch(static_cast<const uint8_t*>(c->img) + static_cast<size_t>(b0) * (c->img_bytes / c->cfg.batch),
                              c->cfg.input_dtype == 1, n, c->cfg.height, c->cfg.width, u.hi, u.lo, u.H, u.W, st);
  }).bytes = static_cast<double>(c->img_bytes) + static_cast<double>(c->stem_u.elems()) * esz;
  // use_gn (nn.py:859-862, 474-477): every backbone conv is a plain conv followed by GroupNorm steps that carry the ReLU
  // and the residual; with BatchNorm the norm, ReLU and residual are in the conv epilogue
  const bool gn = cfg.use_gn != 0;
  // ResNeXt 32x4d blocks (nn.py:524-549, chosen at :864-868): conv1 / conv2 at twice the width, conv2 grouped; the block
  // has no squeeze-excite branch, so use_resnext overrides use_se
  const bool rx = cfg.use_resnext != 0;
  // basic blocks (--resnet34 / --resnet18, nn.py:439-456): block_func is reassigned to ResNeXt after them, so use_resnext
  // wins (nn.py:864-868)
  const bool basic = c->ext.use_basic_block != 0 && !rx;
  const bool se = cfg.use_se != 0 && !rx && !basic;   // squeeze-excite bottlenecks (nn.py:506-519)
  const ConvAffine norm = gn ? kNoAffine : kBatchNorm;
  // conv0 as a 4x1 VALID conv over the packed operand (see stem.cu), BN + ReLU in the epilogue
  {
    Planes view = c->stem_u;
    view.C = 64;                       // one GEMM pixel = 4 consecutive operand pixels
    ConvDesc d = conv_desc(4, 64);
    d.S = 1;
    d.in_H = c->c1h + 3; d.in_W = c->c1w;
    d.in_ld = 16;
    d.relu = !gn;
    add_conv(P, 0, "conv0", view, d, norm, c->c1, nullptr, kStem);
    if (gn && add_gn(P, 0, "conv0/gn", c->c1, c->c1h, c->c1w, 0, 0, nullptr, 0, true)) return -1;
  }
  add_batch_step(P, 0, kStepMaxpool, "", [c](int b0, int n, cudaStream_t st) {
    const Planes a = c->c1.images(b0, n), p = c->pool.images(b0, n);
    return maxpool_launch(a.hi, a.lo, n, c->c1h, c->c1w, 64, p.hi, p.lo, c->ch[0], c->cw[0], st);
  }).bytes = (static_cast<double>(c->c1.elems()) + c->pool.elems()) * esz;
  P.stages.planes("c1", c->c1);
  P.stages.planes("pool", c->pool);

  // ---- ResNet groups (nn.py:459-588) ----
  Planes cur = c->pool;
  for (int g = 0; g < 4; ++g) {
    const int feat = 64 << g, count = cfg.resnet_blocks[g];
    const int mid = rx ? 2 * feat : feat;   // width of conv1 / conv2
    const int gh = c->ch[g], gw = c->cw[g];
    const int out_c = basic ? feat : feat * 4;   // the blocks' output width (resnet_shortcut's n_out)
    Planes pingpong[2];
    B2_CHECK(P.alloc_planes(pingpong[0], B, gh, gw, out_c), "alloc group out");
    B2_CHECK(P.alloc_planes(pingpong[1], B, gh, gw, out_c), "alloc group out");
    // a bottleneck's conv1 writes t1_first in the first block (the previous group's size), conv2 writes t2_first where it
    // changes the size (stride 2: with dilation its pad row / column must stay zero, which t2 does not keep)
    Planes t1_first, t1, t2, t2_first, sc;
    if (!basic) B2_CHECK(P.alloc_planes(t1_first, B, cur.H, cur.W, mid), "alloc t1");
    B2_CHECK(P.alloc_planes(t1, B, gh, gw, mid), "alloc t1");   // a basic block's conv1 output is gh x gw at any stride
    if (!basic) {
      B2_CHECK(P.alloc_planes(t2, B, gh, gw, mid), "alloc t2");
      B2_CHECK(P.alloc_planes(t2_first, B, gh, gw, mid), "alloc t2");
    }
    B2_CHECK(P.alloc_planes(sc, B, gh, gw, out_c), "alloc shortcut");
    for (int i = 0; i < count; ++i) {
      const std::string p = "group" + std::to_string(g) + "/block" + std::to_string(i);
      const int stride = (g > 0 && i == 0) ? 2 : 1;
      const Planes& out = pingpong[i & 1];
      if (basic) {
        if (add_basic_block(P, p, cur, stride, BlockBufs{t1, Planes(), sc, out}, gn)) return -1;
      } else {
        const bool in_last3 = i >= count - 3;
        const int dil = (g == 3 && cfg.use_dilations && in_last3) ? 2 : 1;
        // use_deformable (nn.py:470-486, 577-581): a stride-2 block among the last 3 of its group; the ResNeXt block has
        // no deformable branch
        const bool deform = cfg.use_deformable != 0 && !rx && stride == 2 && in_last3;
        const BlockBufs bufs{i == 0 ? t1_first : t1, stride == 2 ? t2_first : t2, sc, out};
        if (add_bottleneck(P, p, cur, stride, dil, bufs, gn, se, rx, deform)) return -1;
      }
      cur = out;
    }
    c->cfeat[g] = cur;
    P.stages.planes("c" + std::to_string(g + 2), cur);
  }

  // ---- FPN (nn.py:947-1014), phase 1 ----
  const int nc = cfg.fpn_num_channel;
  for (int i = 3; i >= 0; --i) {
    B2_CHECK(P.alloc_planes(c->lat[i], B, c->ch[i], c->cw[i], nc), "alloc lateral");
    const std::string nm = "fpn/lateral_1x1_c" + std::to_string(i + 2);
    // use_gn: GroupNorm of the lateral before the top-down sum (gn_c*, nn.py:987-990); its apply step does the
    // nearest-2x upsample-add that the conv epilogue does otherwise
    const Planes* up = i < 3 ? &c->lat[i + 1] : nullptr;
    ConvDesc d = conv_desc(1, nc);
    d.res_shift = 1;
    add_conv(P, 1, nm, c->cfeat[i], d, kBias, c->lat[i], gn ? nullptr : up);
    if (gn && add_gn(P, 1, "fpn/gn_c" + std::to_string(i + 2), c->lat[i], c->ch[i], c->cw[i], 0, 0, up, 1, false))
      return -1;
  }
  for (int i = 0; i < 4; ++i) {
    B2_CHECK(P.alloc_planes(c->pfeat[i], B, c->pfh[i], c->pfw[i], nc), "alloc p");
    const std::string nm = "fpn/posthoc_3x3_p" + std::to_string(i + 2);
    ConvDesc d = conv_desc(3, nc);
    pad_all(d, 1);
    add_conv(P, 1, nm, c->lat[i], d, kBias, c->pfeat[i]);
    // gn_p* (nn.py:1007-1009) over the whole, uncropped level; p6 below subsamples the normalised p5
    if (gn && add_gn(P, 1, "fpn/gn_p" + std::to_string(i + 2), c->pfeat[i], c->pfh[i], c->pfw[i], 0, 0, nullptr, 0, false))
      return -1;
    P.stages.planes("p" + std::to_string(i + 2), c->pfeat[i]);
  }
  B2_CHECK(P.alloc_planes(c->pfeat[4], B, c->pfh[4], c->pfw[4], nc), "alloc p6");
  add_batch_step(P, 1, kStepP6Subsample, "", [c](int b0, int n, cudaStream_t st) {
    const Planes p5 = c->pfeat[3].images(b0, n), p6 = c->pfeat[4].images(b0, n);
    const size_t total = static_cast<size_t>(n) * p6.H * p6.W * (p6.C / 8);
    subsample2_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(p5.hi, p5.lo, n, p5.H, p5.W, p5.C, p6.hi,
                                                                                   p6.lo, p6.H, p6.W);
    B2_CUDA(cudaGetLastError());
    return 0;
  });
  P.stages.planes("p6", c->pfeat[4]);

  // ---- RPN head (models.py:979-1009), phase 2; class+box 1x1 fused into one N=15 GEMM ----
  for (int i = 0; i < 5; ++i) {
    B2_CHECK(P.alloc_planes(c->rpn_h[i], B, c->ph[i], c->pw[i], nc), "alloc rpn hidden");
    ConvDesc d = conv_desc(3, nc);
    d.in_H = c->ph[i]; d.in_W = c->pw[i];   // the cropped level
    pad_all(d, 1);
    d.relu = 1;
    add_conv(P, 2, "rpn/conv0", c->pfeat[i], d, kBias, c->rpn_h[i]);
    c->rpn_out[i] = P.arena.alloc<float>(static_cast<size_t>(B) * c->ph[i] * c->pw[i] * 16 + 16 * 128);
    add_conv_f32(P, 2, "rpn/classbox", c->rpn_h[i], conv_desc(1, 15), kBias, c->rpn_out[i], 16, kRpnOut);
    P.stages.raw("rpn_l" + std::to_string(i), c->rpn_out[i], Stage::kF32, B, c->ph[i], c->pw[i], 16);
  }

  // ---- proposals (phase 3) ----
  RpnParams& rp = c->rpn;
  memset(&rp, 0, sizeof(rp));
  const int K = cfg.rpn_topk;
  for (int i = 0; i < 5; ++i) {
    rp.logits[i] = c->rpn_out[i];
    rp.h[i] = c->ph[i];
    rp.w[i] = c->pw[i];
    rp.stride[i] = cfg.anchor_strides[i];
    cell_anchors(cfg.anchor_strides[i], cfg.anchor_sizes[i], cfg.anchor_ratios, rp.cell[i]);
  }
  rp.B = B; rp.topk = K;
  rp.img_h = static_cast<float>(H); rp.img_w = static_cast<float>(W);
  rp.decode_clip = logf(cfg.max_size / 16.0f);
  {
    const double dc = log(static_cast<double>(cfg.max_size) / 16.0);   // np.log in float64, cast at use
    rp.decode_clip = static_cast<float>(dc);
  }
  rp.min_size = cfg.rpn_min_size;
  rp.multi = cfg.multi_semantics;
  rp.nms_thr = cfg.rpn_nms_thres;
  rp.lvl_boxes = P.arena.alloc<float>(static_cast<size_t>(B) * 5 * K * 4);
  rp.lvl_scores = P.arena.alloc<float>(static_cast<size_t>(B) * 5 * K);
  rp.lvl_count = P.arena.alloc<int>(B * 5);
  rp.prop_boxes = P.arena.alloc<float>(static_cast<size_t>(B) * K * 4);
  rp.prop_scores = P.arena.alloc<float>(static_cast<size_t>(B) * K);
  rp.prop_count = P.arena.alloc<int>(B);
  add_batch_step(P, 3, kStepRpnProposals, "", [c](int, int, cudaStream_t st) { return rpn_proposals_launch(c->rpn, st); }, 2);
  P.stages.raw("lvl_boxes", rp.lvl_boxes, Stage::kF32, B, 5, K, 4);
  P.stages.raw("lvl_scores", rp.lvl_scores, Stage::kF32, B, 5, K, 1);
  P.stages.raw("lvl_count", rp.lvl_count, Stage::kI32, B, 5, 1, 1);
  P.stages.raw("proposal_boxes", rp.prop_boxes, Stage::kF32, B, K, 4, 1);
  P.stages.raw("proposal_scores", rp.prop_scores, Stage::kF32, B, K, 1, 1);
  P.stages.raw("proposal_count", rp.prop_count, Stage::kI32, B, 1, 1, 1);

  // ---- ROIAlign of the proposals (phase 4) ----
  const int M = B * K;
  const int Mpad = (M + 127) / 128 * 128;
  B2_CHECK(P.alloc_planes(c->roi_feat, 1, 1, Mpad, 49 * nc), "alloc roi feat");
  RoiAlignParams& r1 = c->roi1;
  memset(&r1, 0, sizeof(r1));
  for (int i = 0; i < 4; ++i) {
    r1.feat_hi[i] = c->pfeat[i].hi;
    r1.feat_lo[i] = c->pfeat[i].lo;
    r1.H[i] = c->ph[i]; r1.W[i] = c->pw[i];
    r1.pitch_H[i] = c->pfh[i]; r1.pitch_W[i] = c->pfw[i];
    r1.inv_stride[i] = 1.0f / cfg.anchor_strides[i];
  }
  r1.C = nc; r1.B = B; r1.rois_per_image = K;
  r1.boxes = rp.prop_boxes; r1.count = rp.prop_count;
  r1.out_hi = c->roi_feat.hi; r1.out_lo = c->roi_feat.lo; r1.out_nchw = nullptr;
  add_batch_step(P, 4, kStepRoialignProposals, "", [c](int, int, cudaStream_t st) { return roialign_launch(c->roi1, st); });
  P.stages.planes("roi_feat", c->roi_feat);

  // ---- box head (models.py:1030-1108), phase 5: fc6, fc7, class+box outputs fused (N = 5*num_class) ----
  const int dim = cfg.fc_head_dim;
  B2_CHECK(dim % 64 == 0, "b2_create: fc_head_dim must be a multiple of 64");
  const int hd = cfg.conv_head_dim;
  if (hd <= 0) {
    B2_CHECK(P.alloc_rows(c->fc6, M, dim), "alloc fc6");
    B2_CHECK(P.alloc_rows(c->fc7, M, dim), "alloc fc7");
  }
  // the classes the box head outputs and the post-processing sees: with use_partial_classes the background and the
  // selected classes (models.py:807-828, num_class = len(ids) + 1); cfg.num_class stays the checkpoint's
  const int ncls = c->ext2.num_partial_classes > 0 ? c->ext2.num_partial_classes + 1 : cfg.num_class;
  const int nout = ncls + (cfg.class_agnostic ? 4 : ncls * 4);
  const int ldo = (nout + 15) / 16 * 16;
  c->head_logits = P.arena.alloc<float>(static_cast<size_t>(Mpad) * ldo);
  Planes rf = c->roi_feat; rf.W = M;
  ConvDesc fc = conv_desc(1, dim);   // fc6 / fc7 / the conv head's fc: dense + bias + ReLU
  fc.relu = 1;
  // use_att_frcnn_head (models.py:1064-1089): the outputs read hidden + relu(att_trans(the bin sums of the raw ROIAlign
  // features)), after the conv head or the relation modules; the class-agnostic heads (models.py:1126-1170) have no
  // attention branch
  const bool att = c->ext3.use_att_frcnn_head != 0 && !cfg.class_agnostic;
  if (att)
    B2_CHECK(P.alloc_rows(c->att_pool, M, nc) && P.alloc_rows(c->att, M, dim) && P.alloc_rows(c->att_sum, M, dim),
             "alloc attention head");
  Planes head_in;   // the rows fastrcnn/outputs reads
  const ConvLayer *head_fc6 = nullptr, *head_fc7 = nullptr;   // the 2fc head's layers (the small-object branch runs them)
  auto attend = [&](const Planes& hidden) {
    head_in = att ? c->att_sum : hidden;
    return att ? add_att_head(P, c->roi_feat, nc, hidden, c->att_pool, c->att, c->att_sum) : 0;
  };
  if (hd > 0) {
    // conv_frcnn_head (models.py:1110-1125), use_conv_frcnn_head: 4 x [conv 3x3 SAME + bias + ReLU, then GroupNorm per ROI
    // if use_gn] on the [M][7][7] ROI maps (the ROIAlign rows are already (y*7+x)*256+c per ROI: M small images, as in the
    // mask head), then dense "fc" + ReLU over the NCHW flatten (fc6's row permutation with conv_head_dim channels)
    B2_CHECK(hd % 64 == 0 && hd <= 2048 && (!gn || 2048 % hd == 0),
             "b2_create: conv_head_dim must be a multiple of 64 (a power of two from 64 to 2048 with use_gn)");
    B2_CHECK(P.alloc_planes(c->head_a, Mpad, 7, 7, hd) && P.alloc_planes(c->head_b, Mpad, 7, 7, hd), "alloc conv head");
    B2_CHECK(P.alloc_rows(c->fc6, M, dim), "alloc fc");
    Planes rf7 = c->roi_feat; rf7.B = M; rf7.H = 7; rf7.W = 7; rf7.C = nc;
    Planes ha = c->head_a; ha.B = M;
    Planes hb = c->head_b; hb.B = M;
    Planes cur_h = rf7;
    ConvDesc d = conv_desc(3, hd);
    pad_all(d, 1);
    d.relu = 1;
    for (int k = 0; k < 4; ++k) {
      const Planes& o = (k & 1) ? hb : ha;
      add_conv(P, 5, "fastrcnn/conv" + std::to_string(k), cur_h, d, kBias, o);
      if (gn && add_gn(P, 5, "fastrcnn/gn" + std::to_string(k), o, 7, 7, 0, 0, nullptr, 0, false, true)) return -1;
      cur_h = o;
    }
    Planes flat = cur_h; flat.B = 1; flat.H = 1; flat.W = M; flat.C = 49 * hd;
    const Planes& f = c->fc6;
    add_conv(P, 5, "fastrcnn/fc", flat, fc, kBias, f, nullptr, kFc6);
    if (attend(f)) return -1;
    add_conv_f32(P, 5, "fastrcnn/outputs", head_in, conv_desc(1, nout), kBias, c->head_logits, ldo, kHeadOut);
    P.stages.planes("fc", f);
  } else {
    const Planes &f6 = c->fc6, &f7 = c->fc7;
    // add_relation_nn (models.py:1044-1054): fc7 reads relu(fc6) + RM_r1, the outputs read relu(fc7) + RM_r2
    const bool rel = cfg.add_relation_nn != 0;
    Planes h1 = f6, h2 = f7;
    if (rel) {
      B2_CHECK(dim % 64 == 0, "b2_create: add_relation_nn needs fc_head_dim a multiple of 64");
      B2_CHECK(P.alloc_rows(c->rm1, M, dim) && P.alloc_rows(c->rm2, M, dim), "alloc relation sums");
      h1 = c->rm1;
      h2 = c->rm2;
    }
    head_fc6 = add_conv(P, 5, "fastrcnn/fc6", rf, fc, kBias, f6, nullptr, kFc6);
    if (rel && add_relation(P, "fastrcnn/RM_r1", B, K, dim, rp.prop_boxes, rp.prop_count, f6, h1)) return -1;
    head_fc7 = add_conv(P, 5, "fastrcnn/fc7", h1, fc, kBias, f7, nullptr, kDense);
    if (rel && add_relation(P, "fastrcnn/RM_r2", B, K, dim, rp.prop_boxes, rp.prop_count, f7, h2)) return -1;
    if (attend(h2)) return -1;
    add_conv_f32(P, 5, "fastrcnn/outputs", head_in, conv_desc(1, nout), kBias, c->head_logits, ldo, kHeadOut);
    P.stages.planes("fc6", f6);
    P.stages.planes("fc7", f7);
    if (rel) {
      P.stages.planes("rm_r1", h1);
      P.stages.planes("rm_r2", h2);
    }
  }
  P.stages.raw("head_logits", c->head_logits, Stage::kF32, B, K, ldo, 1);

  // ---- post-processing (phase 6) ----
  HeadPostParams& hp = c->post;
  memset(&hp, 0, sizeof(hp));
  const int nc1 = ncls - 1, R = cfg.result_per_im;
  hp.logits = c->head_logits; hp.ld = ldo; hp.num_class = ncls; hp.B = B; hp.rois_per_image = K;
  hp.class_agnostic = cfg.class_agnostic;
  hp.rois = rp.prop_boxes; hp.roi_count = rp.prop_count;
  for (int i = 0; i < 4; ++i) hp.reg_w[i] = cfg.bbox_reg_weights[i];
  hp.decode_clip = static_cast<float>(log(1333.0 / 16.0));   // decode_bbox_target default (nn.py:1518)
  hp.img_h = static_cast<float>(H); hp.img_w = static_cast<float>(W);
  // batch graph: combined_non_max_suppression is called without a score threshold (models.py:2959-2965)
  hp.score_thresh = cfg.multi_semantics ? -INFINITY : cfg.result_score_thres;
  hp.nms_thr = cfg.fastrcnn_nms_iou_thres;
  hp.max_per_class = R; hp.max_total = R;
  hp.probs = P.arena.alloc<float>(static_cast<size_t>(M) * ncls);
  hp.dec_boxes = P.arena.alloc<float>(static_cast<size_t>(M) * nc1 * 4);
  hp.cls_keep = P.arena.alloc<int>(static_cast<size_t>(B) * nc1 * R);
  hp.cls_count = P.arena.alloc<int>(B * nc1);
  hp.final_boxes = P.arena.alloc<float>(static_cast<size_t>(B) * R * 4);
  hp.final_probs = P.arena.alloc<float>(static_cast<size_t>(B) * R);
  hp.final_labels = P.arena.alloc<int>(static_cast<size_t>(B) * R);
  hp.final_count = P.arena.alloc<int>(B);
  // use_bg_score (models.py:1263-1270): the single-image graph's fastrcnn_predictions drops background-argmax rows; the
  // batch graph's combined NMS (models.py:2924-2976) has no such filter
  if (c->ext5.use_bg_score && !cfg.multi_semantics) {
    hp.bg_rank = P.arena.alloc<int>(static_cast<size_t>(M));
    B2_CHECK(hp.bg_rank, "out of device memory (background filter)");
    P.stages.raw("bg_rank", hp.bg_rank, Stage::kI32, B, K, 1, 1);
  }
  add_batch_step(P, 6, kStepHeadPost, "", [c](int, int, cudaStream_t st) { return head_post_launch(c->post, st); },
                 hp.bg_rank ? 4 : 3);
  P.stages.raw("probs", hp.probs, Stage::kF32, B, K, ncls, 1);
  P.stages.raw("dec_boxes", hp.dec_boxes, Stage::kF32, B, K, nc1, 4);
  P.stages.raw("final_boxes", hp.final_boxes, Stage::kF32, B, R, 4, 1);
  P.stages.raw("final_probs", hp.final_probs, Stage::kF32, B, R, 1, 1);
  P.stages.raw("final_labels", hp.final_labels, Stage::kI32, B, R, 1, 1);
  P.stages.raw("final_count", hp.final_count, Stage::kI32, B, 1, 1, 1);
  if (c->ext4.use_small_object_head && add_small_objects(c, head_fc6, head_fc7)) return -1;

  // ---- fpn_box_feat: ROIAlign of the final boxes (models.py:972-973), phase 7 ----
  c->box_feat = P.arena.alloc<float>(static_cast<size_t>(B) * R * nc * 49);
  c->box_feat_pooled = P.arena.alloc<float>(static_cast<size_t>(B) * R * nc);
  RoiAlignParams& r2 = c->roi2;
  r2 = r1;
  r2.rois_per_image = R;
  r2.boxes = hp.final_boxes; r2.count = hp.final_count;
  r2.out_hi = nullptr; r2.out_lo = nullptr; r2.out_nchw = c->box_feat;
  add_batch_step(P, 7, kStepRoialignFinal, "", [c](int, int, cudaStream_t st) {
    if (roialign_launch(c->roi2, st)) return -1;
    const int rows = c->cfg.batch * c->cfg.result_per_im;
    pool_feat_kernel<<<(rows * c->cfg.fpn_num_channel + 255) / 256, 256, 0, st>>>(c->box_feat, rows, c->cfg.fpn_num_channel,
                                                                                   c->box_feat_pooled);
    B2_CUDA(cudaGetLastError());
    return 0;
  }, 2);
  P.stages.raw("fpn_box_feat", c->box_feat, Stage::kF32, static_cast<int64_t>(B) * R, nc, 7, 7);

  // ---- mask head (models.py:934-961, 1173-1199), phase 7, only with cfg.add_mask ----
  // ROIAlign 14 of the final boxes, fcn0..3, the deconv, the class conv and the own-class sigmoid (add_mask_head); the
  // layers ping-pong between two buffers
  if (cfg.add_mask) {
    const int MR = B * R, md = 256;                  // mrcnn_head_dim (obj_detect_tracking.py:324)
    B2_CHECK(P.alloc_planes(c->mask_a, MR, 14, 14, md), "alloc mask head a");
    B2_CHECK(P.alloc_planes(c->mask_b, MR, 14, 14, md), "alloc mask head b");
    B2_CHECK(P.alloc_planes(c->mask_up, MR, 14, 14, 4 * md), "alloc mask head deconv");
    RoiAlignParams r3 = r1;
    r3.rois_per_image = R;
    r3.boxes = hp.final_boxes; r3.count = hp.final_count;
    c->mask_ld = mask_logits_ld(cfg.num_class);
    c->mask_logits = P.arena.alloc<float>(mask_logits_rows(MR) * c->mask_ld);
    c->final_masks = P.arena.alloc<float>(static_cast<size_t>(MR) * 784);
    const MaskBufs mb = {c->mask_a, {c->mask_b, c->mask_a, c->mask_b, c->mask_a}, c->mask_up};
    if (add_mask_head(P, r3, cfg.num_class, mb, hp.final_labels, c->mask_logits, c->final_masks)) return -1;
    P.stages.raw("mask_logits", c->mask_logits, Stage::kF32, MR, 196 * 4, c->mask_ld, 1);
    P.stages.raw("final_masks", c->final_masks, Stage::kF32, B, R, 28, 28);
  }

  // ---- fpn_feature (models.py:517-518): b2_fpn_feature's output, outside the per-frame plan ----
  c->fpn_feat = P.arena.alloc<float>(static_cast<size_t>(B) * 49 * nc);
  B2_CHECK(c->fpn_feat != nullptr, "out of device memory (fpn_feature)");

  // ---- tensor-core plans ----
  return plan_layers(P, c->num_sms);
}

// The phases of `mask` with phases 0-2 forked over nsplit streams (also valid inside a stream capture: the side streams
// join the capture through the fork event and rejoin before the proposals).
int enqueue_dual(b2_ctx* c, unsigned mask) {
  B2_CUDA(cudaEventRecord(c->fork_ev, c->stream));
  for (int h = 1; h < c->plan.nsplit; ++h) B2_CUDA(cudaStreamWaitEvent(c->side_stream[h - 1], c->fork_ev, 0));
  for (const Step& s : c->plan.steps) {
    if (s.phase > 2 || !((mask >> s.phase) & 1u)) continue;
    for (int h = 0; h < c->plan.nsplit; ++h)
      if (s.parts[h](h == 0 ? c->stream : c->side_stream[h - 1])) return -1;
  }
  for (int h = 1; h < c->plan.nsplit; ++h) {
    B2_CUDA(cudaEventRecord(c->join_ev[h - 1], c->side_stream[h - 1]));
    B2_CUDA(cudaStreamWaitEvent(c->stream, c->join_ev[h - 1], 0));
  }
  return run_steps(c->plan.steps, mask & ~0x7u, c->stream);
}

int enqueue(b2_ctx* c, int mask, bool with_events) {
  if (c->plan.dual && !with_events && mask == B2_PHASE_ALL) return enqueue_dual(c, B2_PHASE_ALL);
  if (!with_events) return run_steps(c->plan.steps, mask, c->stream);
  B2_CUDA(cudaEventRecord(c->ev[0], c->stream));
  int last = -1;
  for (const Step& s : c->plan.steps) {
    if (!(mask & (1 << s.phase))) continue;
    if (last >= 0 && s.phase != last) B2_CUDA(cudaEventRecord(c->ev[last + 1], c->stream));
    if (s.run(c->stream)) return -1;
    last = s.phase;
  }
  if (last >= 0) B2_CUDA(cudaEventRecord(c->ev[last + 1], c->stream));
  return 0;
}

int fpn_feature_launch(b2_ctx* c) {
  const Planes& p5 = c->pfeat[3];
  const int total = p5.B * 49 * (p5.C / 8);
  fpn_feature_kernel<<<(total + 255) / 256, 256, 0, c->stream>>>(p5.hi, p5.lo, p5.B, p5.H, p5.W, p5.C, c->pfh[3], c->pfw[3],
                                                                  tf_resize_scale(c->pfh[3], 7), tf_resize_scale(c->pfw[3], 7),
                                                                  c->fpn_feat);
  B2_CUDA(cudaGetLastError());
  return 0;
}

// The backbone-only pass of b2_fpn_feature: phases 0-1, forked over the batch parts as in a full pass, then the resize.
int enqueue_feature(b2_ctx* c) {
  const unsigned mask = B2_PHASE_BACKBONE | B2_PHASE_FPN;
  if (c->plan.dual ? enqueue_dual(c, mask) : run_steps(c->plan.steps, mask, c->stream)) return -1;
  return fpn_feature_launch(c);
}

}  // namespace

// =================================================================================================
extern "C" {

int b2_create(b2_ctx** out, int device, const b2_config* cfg) { return b2_create_ex(out, device, cfg, nullptr); }

int b2_create_ex(b2_ctx** out, int device, const b2_config* cfg, const b2_config_ext* ext) {
  return b2_create_ex2(out, device, cfg, ext, nullptr);
}

int b2_create_ex2(b2_ctx** out, int device, const b2_config* cfg, const b2_config_ext* ext, const b2_config_ext2* ext2) {
  return b2_create_ex3(out, device, cfg, ext, ext2, nullptr);
}

int b2_create_ex3(b2_ctx** out, int device, const b2_config* cfg, const b2_config_ext* ext, const b2_config_ext2* ext2,
                  const b2_config_ext3* ext3) {
  return b2_create_ex4(out, device, cfg, ext, ext2, ext3, nullptr);
}

int b2_create_ex4(b2_ctx** out, int device, const b2_config* cfg, const b2_config_ext* ext, const b2_config_ext2* ext2,
                  const b2_config_ext3* ext3, const b2_config_ext4* ext4) {
  return b2_create_ex5(out, device, cfg, ext, ext2, ext3, ext4, nullptr);
}

int b2_create_ex5(b2_ctx** out, int device, const b2_config* cfg, const b2_config_ext* ext, const b2_config_ext2* ext2,
                  const b2_config_ext3* ext3, const b2_config_ext4* ext4, const b2_config_ext5* ext5) {
  B2_CHECK(out && cfg, "b2_create: null argument");
  *out = nullptr;
  std::unique_ptr<b2_ctx> c(new b2_ctx());
  c->cfg = *cfg;
  memset(&c->ext, 0, sizeof(c->ext));
  if (ext) c->ext = *ext;
  memset(&c->ext2, 0, sizeof(c->ext2));
  if (ext2) c->ext2 = *ext2;
  memset(&c->ext3, 0, sizeof(c->ext3));
  if (ext3) c->ext3 = *ext3;
  memset(&c->ext4, 0, sizeof(c->ext4));
  if (ext4) c->ext4 = *ext4;
  memset(&c->ext5, 0, sizeof(c->ext5));
  if (ext5) c->ext5 = *ext5;
  const int np = c->ext2.num_partial_classes;
  B2_CHECK(np >= 0 && np <= cfg->num_class - 1 && np <= 80,
           "b2_create: num_partial_classes must be 0 (off) or 1 .. min(num_class - 1, 80) (num_class " +
               std::to_string(cfg->num_class) + "), got " + std::to_string(np));
  for (int i = 0; i < np; ++i) {
    const int id = c->ext2.partial_class_ids[i];
    B2_CHECK(id >= 1 && id <= cfg->num_class - 1, "b2_create: partial_class_ids[" + std::to_string(i) + "] = " +
                                                      std::to_string(id) + " is not a class id in 1 .. num_class - 1");
    for (int j = 0; j < i; ++j)
      B2_CHECK(c->ext2.partial_class_ids[j] != id, "b2_create: class id " + std::to_string(id) +
                                                      " appears twice in partial_class_ids");
  }
  const b2_config_ext4& so = c->ext4;
  if (so.use_small_object_head) {
    const std::string who = "b2_create: use_small_object_head ";
    B2_CHECK(!cfg->class_agnostic, who + "cannot be combined with use_frcnn_class_agnostic: the reference's decode reshapes "
                                         "[N,1,4] box logits against [N,num_class-1,4] anchors and fails");
    B2_CHECK(np == 0, who + "cannot be combined with use_partial_classes: the branch reads the full head's class columns");
    B2_CHECK(cfg->conv_head_dim <= 0, who + "cannot be combined with use_conv_frcnn_head: the branch would need its own "
                                             "fc6 / fc7 next to fastrcnn/fc");
    B2_CHECK(cfg->batch == 1 && !cfg->multi_semantics, who + "needs batch 1 and the single-image graph: the batch graph "
                                                             "(Mask_RCNN_FPN_multi) has no small-object branch");
    const int C = so.num_small_objects;
    B2_CHECK(C >= 1 && C <= cfg->num_class - 1 && C <= 80, who + "num_small_objects must be 1 .. min(num_class - 1, 80), got " +
                                                              std::to_string(C));
    for (int i = 0; i < C; ++i) {
      const int id = so.small_object_class_ids[i];
      B2_CHECK(id >= 1 && id <= cfg->num_class - 1, who + "small_object_class_ids[" + std::to_string(i) + "] = " +
                                                        std::to_string(id) + " is not a class id in 1 .. num_class - 1");
      for (int j = 0; j < i; ++j)
        B2_CHECK(so.small_object_class_ids[j] != id, who + "class id " + std::to_string(id) + " appears twice");
    }
    if (so.use_so_association) {
      B2_CHECK(so.so_person_class_id >= 1 && so.so_person_class_id <= cfg->num_class - 1,
               who + "so_person_class_id " + std::to_string(so.so_person_class_id) + " is not a class id in 1 .. num_class - 1");
      B2_CHECK(so.so_person_topk >= 1 && so.so_person_topk <= 1024,
               who + "so_person_topk must be 1 .. 1024, got " + std::to_string(so.so_person_topk));
    }
  }
  c->device = device;
  c->plan.split = cfg->precision == 1;
  if (open_device(device, "b2_create", &c->num_sms, &c->stream)) return -1;
  for (int i = 0; i <= NPHASE; ++i) B2_CUDA(cudaEventCreate(&c->ev[i]));
  memset(c->phase_ms, 0, sizeof(c->phase_ms));
  if (build_plan(c.get())) {
    b2_destroy(c.release());
    return -1;
  }
  if (c->plan.dual) {
    B2_CUDA(cudaEventCreateWithFlags(&c->fork_ev, cudaEventDisableTiming));
    for (int h = 1; h < c->plan.nsplit; ++h) {
      B2_CUDA(cudaStreamCreateWithFlags(&c->side_stream[h - 1], cudaStreamNonBlocking));
      B2_CUDA(cudaEventCreateWithFlags(&c->join_ev[h - 1], cudaEventDisableTiming));
    }
  }
  B2_CUDA(cudaDeviceSynchronize());
  *out = c.release();
  return 0;
}

void b2_destroy(b2_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  if (c->graph) cudaGraphExecDestroy(c->graph);
  if (c->feat_graph) cudaGraphExecDestroy(c->feat_graph);
  if (c->fork_ev) cudaEventDestroy(c->fork_ev);
  for (int h = 0; h < 7; ++h) {
    if (c->join_ev[h]) cudaEventDestroy(c->join_ev[h]);
    if (c->side_stream[h]) cudaStreamDestroy(c->side_stream[h]);
  }
  if (c->raw_frames) cudaFree(c->raw_frames);
  if (c->h_range) cudaFreeHost(c->h_range);
  for (int i = 0; i <= NPHASE; ++i)
    if (c->ev[i]) cudaEventDestroy(c->ev[i]);
  for (int i = 0; i < 2; ++i) {
    if (c->h2d_done[i]) cudaEventDestroy(c->h2d_done[i]);
    if (c->staged_free[i]) cudaEventDestroy(c->staged_free[i]);
    if (c->out_done[i]) cudaEventDestroy(c->out_done[i]);
    if (c->pass_done[i]) cudaEventDestroy(c->pass_done[i]);
  }
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  if (c->down_stream) cudaStreamDestroy(c->down_stream);
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;   // plans, then the arena's device memory
}

int b2_load_weights(b2_ctx* c, const char* const* names, const float* const* data, const int64_t* numel, int n) {
  B2_CHECK(c && names && data && numel, "b2_load_weights: null argument");
  B2_CUDA(cudaSetDevice(c->device));
  const WeightSet ws(names, data, numel, n);
  if (load_weights(c->plan, ws, c->cfg.num_class, c->stream, c->ext2.partial_class_ids, c->ext2.num_partial_classes))
    return -1;
  c->weights_loaded = true;
  return 0;
}

static int range_failed(b2_ctx* c, int idx);

// Waits for the stream and fails when the pass left the fp16-plane range (synchronous calls).
static int sync_range(b2_ctx* c) {
  B2_CUDA(cudaMemcpyAsync(&c->h_range[2], c->plan.range_flag, sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
  B2_CUDA(cudaStreamSynchronize(c->stream));
  return range_failed(c, 2);
}

int b2_run_phases(b2_ctx* c, int mask) {
  B2_CHECK(c, "b2_run_phases: null ctx");
  B2_CUDA(cudaSetDevice(c->device));
  B2_CHECK(c->weights_loaded, "b2_run_phases: weights not loaded");
  if (enqueue(c, mask, true) || sync_range(c)) return -1;
  int last = -1;
  for (int ph = 0; ph < NPHASE; ++ph) {
    c->phase_ms[ph] = 0.f;
    if (!(mask & (1 << ph))) continue;
    bool any = false;
    for (const auto& s : c->plan.steps) any = any || s.phase == ph;
    if (!any) continue;
    cudaEventElapsedTime(&c->phase_ms[ph], c->ev[last < 0 ? 0 : last + 1], c->ev[ph + 1]);
    last = ph;
  }
  return 0;
}

int b2_phase_times(b2_ctx* c, float ms[8]) {
  B2_CHECK(c && ms, "b2_phase_times: null argument");
  for (int i = 0; i < NPHASE; ++i) ms[i] = c->phase_ms[i];
  return 0;
}

int b2_kernel_launches(b2_ctx* c) { return c ? total_launches(c->plan.steps) : -1; }

int b2_fpn_feature_launches(b2_ctx* c) {
  if (!c) return -1;
  std::vector<Step> steps;
  for (const Step& s : c->plan.steps)
    if (s.phase <= 1) steps.push_back(s);
  return total_launches(steps) + 1;
}

// Per-step device timing (CUDA events around every launch group, eager mode), averaged over `reps`.
int b2_profile_steps(b2_ctx* c, int reps, float* ms_out, int cap, int* n_out) {
  B2_CHECK(c && ms_out && n_out, "b2_profile_steps: null argument");
  B2_CUDA(cudaSetDevice(c->device));
  B2_CHECK(c->weights_loaded, "b2_profile_steps: weights not loaded");
  return profile_steps(c->plan.steps, c->stream, reps, ms_out, cap, n_out);
}

// Describes step `idx`: name, kind (0 = tensor-core conv/dense), algorithmic FLOPs and HBM bytes
// (each operand read once, output written once, at the stored precision).
int b2_step_info(b2_ctx* c, int idx, char* name, int name_cap, double* flops, double* bytes, int* kind) {
  B2_CHECK(c, "b2_step_info: null argument");
  return step_info(c->plan.steps, idx, name, name_cap, flops, bytes, kind);
}
int b2_num_steps(b2_ctx* c) { return c ? static_cast<int>(c->plan.steps.size()) : -1; }

static int ensure_graph(b2_ctx* c) {
  if (c->graph || !c->cfg.use_cuda_graph) return 0;
  return capture_graph(c->stream, [c] { return enqueue(c, B2_PHASE_ALL, false); }, &c->graph);
}

static int run_all(b2_ctx* c) {
  if (c->cfg.use_cuda_graph) {
    if (ensure_graph(c)) return -1;
    B2_CUDA(cudaGraphLaunch(c->graph, c->stream));
    return 0;
  }
  return enqueue(c, B2_PHASE_ALL, false);
}

// The pass left the representable range of the fp16 activation planes somewhere (the kernel flags |x| > 65504 or NaN at the
// store): the results of this call are not trustworthy.  The flag is cleared so that the next pass is judged on its own.
static int range_failed(b2_ctx* c, int idx) {
  if (c->h_range[idx] == 0) return 0;
  c->h_range[idx] = 0;
  cudaMemsetAsync(c->plan.range_flag, 0, sizeof(unsigned int), c->stream);
  set_error("activation outside the fp16-plane range (|x| > 65504 or NaN) in a convolution output: the weights / input are "
            "not conditioned for the (hi, lo) fp16 representation (DESIGN.md section 3)");
  return -1;
}

static int copy_outputs(b2_ctx* c, float* boxes, float* probs, int32_t* labels, int32_t* valid, float* box_feat,
                        int feat_mode, cudaMemcpyKind kind) {
  const int B = c->cfg.batch, R = c->cfg.result_per_im, C = c->cfg.fpn_num_channel;
  cudaStream_t st = c->stream;
  if (boxes) B2_CUDA(cudaMemcpyAsync(boxes, c->post.final_boxes, sizeof(float) * B * R * 4, kind, st));
  if (probs) B2_CUDA(cudaMemcpyAsync(probs, c->post.final_probs, sizeof(float) * B * R, kind, st));
  if (labels) B2_CUDA(cudaMemcpyAsync(labels, c->post.final_labels, sizeof(int32_t) * B * R, kind, st));
  if (valid) B2_CUDA(cudaMemcpyAsync(valid, c->post.final_count, sizeof(int32_t) * B, kind, st));
  if (box_feat) {
    B2_CHECK(feat_mode >= 0 && feat_mode <= 3, "feat_mode must be 0 (full), 1 (mean), 2 (max) or 3 (spatial)");
    if (feat_mode == 1) {
      B2_CUDA(cudaMemcpyAsync(box_feat, c->box_feat_pooled, sizeof(float) * B * R * C, kind, st));
    } else if (feat_mode >= 2) {
      const int rows = B * R, n = feat_mode == 2 ? rows * C : rows * 49;
      if (!c->box_feat_agg) {
        c->box_feat_agg = c->plan.arena.alloc<float>(static_cast<size_t>(rows) * (C > 49 ? C : 49), /*zero=*/false);   // fully overwritten
        B2_CHECK(c->box_feat_agg != nullptr, "out of device memory (feature aggregation scratch)");
      }
      agg_feat_kernel<<<(n + 255) / 256, 256, 0, st>>>(c->box_feat, rows, C, feat_mode, c->box_feat_agg);
      B2_CUDA(cudaGetLastError());
      B2_CUDA(cudaMemcpyAsync(box_feat, c->box_feat_agg, sizeof(float) * n, kind, st));
    } else {
      B2_CUDA(cudaMemcpyAsync(box_feat, c->box_feat, sizeof(float) * B * R * C * 49, kind, st));
    }
  }
  return 0;
}

int b2_detect(b2_ctx* c, const void* frames_dev, float* boxes, float* probs, int32_t* labels, int32_t* valid,
              float* box_feat, int feat_mode, int sync) {
  B2_CHECK(c, "b2_detect: null ctx");
  B2_CUDA(cudaSetDevice(c->device));
  B2_CHECK(c->weights_loaded, "b2_detect: weights not loaded");
  if (frames_dev && frames_dev != c->img)
    B2_CUDA(cudaMemcpyAsync(c->img, frames_dev, c->img_bytes, cudaMemcpyDeviceToDevice, c->stream));
  if (run_all(c)) return -1;
  if (copy_outputs(c, boxes, probs, labels, valid, box_feat, feat_mode, cudaMemcpyDeviceToDevice)) return -1;
  return sync ? sync_range(c) : 0;
}

int b2_detect_host(b2_ctx* c, const void* frames_host, float* boxes, float* probs, int32_t* labels, int32_t* valid,
                   float* box_feat, int feat_mode) {
  B2_CHECK(c && frames_host, "b2_detect_host: null argument");
  B2_CUDA(cudaSetDevice(c->device));
  B2_CHECK(c->weights_loaded, "b2_detect_host: weights not loaded");
  B2_CUDA(cudaMemcpyAsync(c->img, frames_host, c->img_bytes, cudaMemcpyHostToDevice, c->stream));
  if (run_all(c)) return -1;
  if (copy_outputs(c, boxes, probs, labels, valid, box_feat, feat_mode, cudaMemcpyDeviceToHost)) return -1;
  return sync_range(c);
}

// Frame ingest with the resize on the device (SURVEY 8f rank 1; reference host path: frame.astype("float32") ->
// resizeImage (cv2.resize INTER_LINEAR, nn.py:1540-1545) -> feed, obj_detect_tracking.py:597-608): the uint8 source frames
// cross PCIe (4x fewer bytes than the resized float32 frames the reference feeds, no host resize), resize_u8_to_f32_kernel
// writes the float32 network input.  The caller computes the target size with get_new_hw (nn.py:1548-1560) and creates the
// context for it with input_dtype = 0.
int b2_detect_host_resize(b2_ctx* c, const uint8_t* frames_u8, int src_h, int src_w, float* boxes, float* probs,
                          int32_t* labels, int32_t* valid, float* box_feat, int feat_mode) {
  B2_CHECK(c && frames_u8, "b2_detect_host_resize: null argument");
  B2_CHECK(src_h > 0 && src_w > 0, "b2_detect_host_resize: bad source size");
  B2_CHECK(c->cfg.input_dtype == 0, "b2_detect_host_resize: the context must be created with input_dtype = 0 (float32 frames)");
  B2_CUDA(cudaSetDevice(c->device));
  B2_CHECK(c->weights_loaded, "b2_detect_host_resize: weights not loaded");
  const size_t need = static_cast<size_t>(c->cfg.batch) * src_h * src_w * 3;
  if (need > c->raw_bytes) {
    B2_CUDA(cudaStreamSynchronize(c->stream));
    if (c->raw_frames) B2_CUDA(cudaFree(c->raw_frames));
    c->raw_frames = nullptr;
    c->raw_bytes = 0;
    B2_CUDA(cudaMalloc(&c->raw_frames, need));
    c->raw_bytes = need;
  }
  B2_CUDA(cudaMemcpyAsync(c->raw_frames, frames_u8, need, cudaMemcpyHostToDevice, c->stream));
  if (resize_u8_launch(c->raw_frames, c->cfg.batch, src_h, src_w, static_cast<float*>(c->img), c->cfg.height, c->cfg.width,
                       c->stream)) return -1;
  if (run_all(c)) return -1;
  if (copy_outputs(c, boxes, probs, labels, valid, box_feat, feat_mode, cudaMemcpyDeviceToHost)) return -1;
  return sync_range(c);
}

// Pipelined ingest for streaming drivers (the reference's queue-fed loop, obj_detect_tracking_multi_queuer.py:386-480):
// b2_submit_host enqueues  H2D(frames -> staging[slot]) on a copy stream, then on the compute stream
// staging[slot] -> image, the pass, and the D2H of the results into the caller's (pinned) buffers, and returns without
// waiting; b2_wait(slot) blocks until that slot's results have landed.  With two slots the upload of batch i+1 overlaps
// the pass of batch i.  Host buffers must stay valid (and should be page-locked) until b2_wait returns.
// src_h == 0: frames_host are network-input frames (b2_submit_host).  src_h > 0: uint8 source frames [B, src_h, src_w, 3]
// that the resize kernel turns into the float32 network input on the compute stream (b2_submit_host_resize).
static int submit_impl(b2_ctx* c, const void* frames_host, int src_h, int src_w, float* boxes, float* probs, int32_t* labels,
                       int32_t* valid, float* box_feat, int feat_mode, int slot) {
  B2_CHECK(c && frames_host, "b2_submit_host: null argument");
  B2_CHECK(slot == 0 || slot == 1, "b2_submit_host: slot must be 0 or 1");
  B2_CUDA(cudaSetDevice(c->device));
  B2_CHECK(c->weights_loaded, "b2_submit_host: weights not loaded");
  B2_CHECK(!c->slot_busy[slot], "b2_submit_host: slot still in flight (call b2_wait first)");
  const int B = c->cfg.batch, R = c->cfg.result_per_im, C = c->cfg.fpn_num_channel;
  const size_t nb_boxes = sizeof(float) * B * R * 4, nb_probs = sizeof(float) * B * R, nb_labels = sizeof(int32_t) * B * R;
  const size_t nb_valid = (sizeof(int32_t) * B + 255) / 256 * 256, nb_feat = sizeof(float) * B * R * C * 49;
  if (!c->copy_stream) {
    B2_CUDA(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    B2_CUDA(cudaStreamCreateWithFlags(&c->down_stream, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) {
      c->stage_in[i] = c->plan.arena.alloc<uint8_t>(c->img_bytes, false);
      c->stage_out[i] = c->plan.arena.alloc<uint8_t>(nb_boxes + nb_probs + nb_labels + nb_valid + nb_feat, false);
      B2_CHECK(c->stage_in[i] && c->stage_out[i], "out of device memory (submit staging buffers)");
      B2_CUDA(cudaEventCreateWithFlags(&c->h2d_done[i], cudaEventDisableTiming));
      B2_CUDA(cudaEventCreateWithFlags(&c->staged_free[i], cudaEventDisableTiming));
      B2_CUDA(cudaEventCreateWithFlags(&c->out_done[i], cudaEventDisableTiming));
      B2_CUDA(cudaEventCreateWithFlags(&c->pass_done[i], cudaEventDisableTiming));
      B2_CUDA(cudaEventRecord(c->staged_free[i], c->stream));
    }
    if (c->cfg.use_cuda_graph && ensure_graph(c)) return -1;   // capture before anything is in flight
  }
  const size_t in_bytes = src_h > 0 ? static_cast<size_t>(B) * src_h * src_w * 3 : c->img_bytes;
  B2_CUDA(cudaStreamWaitEvent(c->copy_stream, c->staged_free[slot], 0));      // the previous use of this staging buffer
  B2_CUDA(cudaMemcpyAsync(c->stage_in[slot], frames_host, in_bytes, cudaMemcpyHostToDevice, c->copy_stream));
  B2_CUDA(cudaEventRecord(c->h2d_done[slot], c->copy_stream));
  B2_CUDA(cudaStreamWaitEvent(c->stream, c->h2d_done[slot], 0));
  if (src_h > 0) {
    if (resize_u8_launch(static_cast<const uint8_t*>(c->stage_in[slot]), B, src_h, src_w, static_cast<float*>(c->img),
                         c->cfg.height, c->cfg.width, c->stream)) return -1;
  } else {
    B2_CUDA(cudaMemcpyAsync(c->img, c->stage_in[slot], c->img_bytes, cudaMemcpyDeviceToDevice, c->stream));
  }
  B2_CUDA(cudaEventRecord(c->staged_free[slot], c->stream));
  if (run_all(c)) return -1;
  // results -> this slot's device staging (a few tens of microseconds), then off the compute stream: the download runs
  // on its own stream while the next pass is already executing
  uint8_t* so = c->stage_out[slot];
  uint8_t* d_boxes = so;
  uint8_t* d_probs = d_boxes + nb_boxes;
  uint8_t* d_labels = d_probs + nb_probs;
  uint8_t* d_valid = d_labels + nb_labels;
  uint8_t* d_feat = d_valid + nb_valid;
  const size_t feat_bytes = feat_mode == 1 || feat_mode == 2 ? sizeof(float) * B * R * C
                            : feat_mode == 3 ? sizeof(float) * B * R * 49 : nb_feat;
  if (copy_outputs(c, boxes ? reinterpret_cast<float*>(d_boxes) : nullptr, probs ? reinterpret_cast<float*>(d_probs) : nullptr,
                   labels ? reinterpret_cast<int32_t*>(d_labels) : nullptr, valid ? reinterpret_cast<int32_t*>(d_valid) : nullptr,
                   box_feat ? reinterpret_cast<float*>(d_feat) : nullptr, feat_mode, cudaMemcpyDeviceToDevice)) return -1;
  B2_CUDA(cudaMemcpyAsync(&c->h_range[slot], c->plan.range_flag, sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
  B2_CUDA(cudaEventRecord(c->pass_done[slot], c->stream));
  cudaStream_t ds = c->down_stream;
  B2_CUDA(cudaStreamWaitEvent(ds, c->pass_done[slot], 0));
  if (boxes) B2_CUDA(cudaMemcpyAsync(boxes, d_boxes, nb_boxes, cudaMemcpyDeviceToHost, ds));
  if (probs) B2_CUDA(cudaMemcpyAsync(probs, d_probs, nb_probs, cudaMemcpyDeviceToHost, ds));
  if (labels) B2_CUDA(cudaMemcpyAsync(labels, d_labels, nb_labels, cudaMemcpyDeviceToHost, ds));
  if (valid) B2_CUDA(cudaMemcpyAsync(valid, d_valid, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, ds));
  if (box_feat) B2_CUDA(cudaMemcpyAsync(box_feat, d_feat, feat_bytes, cudaMemcpyDeviceToHost, ds));
  B2_CUDA(cudaEventRecord(c->out_done[slot], ds));
  c->slot_busy[slot] = true;
  return 0;
}

int b2_submit_host(b2_ctx* c, const void* frames_host, float* boxes, float* probs, int32_t* labels, int32_t* valid,
                   float* box_feat, int feat_mode, int slot) {
  return submit_impl(c, frames_host, 0, 0, boxes, probs, labels, valid, box_feat, feat_mode, slot);
}

// The streaming form of b2_detect_host_resize: uint8 source frames in (they must fit the staging buffer, i.e. at most four
// source pixels per network-input pixel), resized on the device, pipelined like b2_submit_host.
int b2_submit_host_resize(b2_ctx* c, const uint8_t* frames_u8, int src_h, int src_w, float* boxes, float* probs,
                          int32_t* labels, int32_t* valid, float* box_feat, int feat_mode, int slot) {
  B2_CHECK(c && src_h > 0 && src_w > 0, "b2_submit_host_resize: bad argument");
  B2_CHECK(c->cfg.input_dtype == 0, "b2_submit_host_resize: the context must be created with input_dtype = 0 (float32 frames)");
  B2_CHECK(static_cast<size_t>(c->cfg.batch) * src_h * src_w * 3 <= c->img_bytes,
           "b2_submit_host_resize: source frames larger than the staging buffer (more than 4 source pixels per input pixel)");
  return submit_impl(c, frames_u8, src_h, src_w, boxes, probs, labels, valid, box_feat, feat_mode, slot);
}

int b2_wait(b2_ctx* c, int slot) {
  B2_CHECK(c && (slot == 0 || slot == 1), "b2_wait: bad argument");
  B2_CUDA(cudaSetDevice(c->device));
  B2_CHECK(c->slot_busy[slot], "b2_wait: nothing was submitted on this slot");
  B2_CUDA(cudaEventSynchronize(c->out_done[slot]));
  c->slot_busy[slot] = false;
  return range_failed(c, slot);
}

// RCNN_FPN_givenbox (models.py:1816-1967; get_model_feat :121-131): features of GIVEN boxes on one frame -- backbone + FPN,
// ROIAlign 7x7 of the boxes on the uncropped p2..p5 (that graph skips slice_feature_and_anchors) and the mean over the
// 7x7 bins (final_box_features [n, 256]).  The context must have batch 1; boxes are processed result_per_im at a time.
int b2_box_features(b2_ctx* c, const void* frame_host, const float* boxes_host, int n, float* feat_host) {
  B2_CHECK(c && frame_host && (n == 0 || (boxes_host && feat_host)), "b2_box_features: null argument");
  B2_CHECK(c->cfg.batch == 1, "b2_box_features: the context must be created with batch 1 (the given-box graph takes one image)");
  B2_CHECK(n >= 0, "b2_box_features: negative box count");
  B2_CUDA(cudaSetDevice(c->device));
  B2_CHECK(c->weights_loaded, "b2_box_features: weights not loaded");
  const int R = c->cfg.result_per_im, C = c->cfg.fpn_num_channel;
  if (!c->given_boxes) {
    c->given_boxes = c->plan.arena.alloc<float>(static_cast<size_t>(R) * 4);
    c->given_count = c->plan.arena.alloc<int>(1);
    c->given_feat = c->plan.arena.alloc<float>(static_cast<size_t>(R) * C * 49);
    c->given_pooled = c->plan.arena.alloc<float>(static_cast<size_t>(R) * C);
    B2_CHECK(c->given_boxes && c->given_count && c->given_feat && c->given_pooled, "out of device memory (given-box buffers)");
    B2_CUDA(cudaDeviceSynchronize());   // the zero fills of alloc() run on the legacy stream
  }
  B2_CUDA(cudaMemcpyAsync(c->img, frame_host, c->img_bytes, cudaMemcpyHostToDevice, c->stream));
  if (enqueue(c, B2_PHASE_BACKBONE | B2_PHASE_FPN, false)) return -1;
  RoiAlignParams rg = c->roi2;
  for (int i = 0; i < 4; ++i) { rg.H[i] = c->pfh[i]; rg.W[i] = c->pfw[i]; }   // uncropped levels
  rg.B = 1; rg.rois_per_image = R;
  rg.boxes = c->given_boxes; rg.count = c->given_count;
  rg.out_hi = nullptr; rg.out_lo = nullptr; rg.out_nchw = c->given_feat; rg.out_res = 7;
  for (int off = 0; off < n; off += R) {
    const int m = n - off < R ? n - off : R;
    B2_CUDA(cudaMemcpyAsync(c->given_boxes, boxes_host + static_cast<size_t>(off) * 4, sizeof(float) * m * 4,
                            cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaMemcpyAsync(c->given_count, &m, sizeof(int), cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));   // `m` lives on this stack frame
    if (roialign_launch(rg, c->stream)) return -1;
    pool_feat_kernel<<<(m * C + 255) / 256, 256, 0, c->stream>>>(c->given_feat, m, C, c->given_pooled);
    B2_CUDA(cudaGetLastError());
    B2_CUDA(cudaMemcpyAsync(feat_host + static_cast<size_t>(off) * C, c->given_pooled, sizeof(float) * m * C,
                            cudaMemcpyDeviceToHost, c->stream));
  }
  B2_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

// final_masks of the last pass (models.py:958-961): [batch][result_per_im][28][28] float32, rows beyond valid[b] are 0.
int b2_get_masks(b2_ctx* c, float* masks_host, int64_t capacity_bytes) {
  B2_CHECK(c && masks_host, "b2_get_masks: null argument");
  B2_CHECK(c->cfg.add_mask && c->final_masks, "b2_get_masks: the context was created without add_mask");
  B2_CUDA(cudaSetDevice(c->device));
  const int64_t bytes = static_cast<int64_t>(c->cfg.batch) * c->cfg.result_per_im * 784 * 4;
  B2_CHECK(capacity_bytes >= bytes, "b2_get_masks: buffer too small");
  B2_CUDA(cudaMemcpyAsync(masks_host, c->final_masks, bytes, cudaMemcpyDeviceToHost, c->stream));
  B2_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

// b2_masks_encode of final_masks rows [0, n) of `image`, read in place (mask_rle.cu) on the context's stream.
int b2_encode_masks(b2_ctx* c, b2_masks* enc, int image, const float* boxes_host, int n, int im_h, int im_w,
                    int64_t* offsets_host, char* bytes_host, int64_t capacity) {
  B2_CHECK(c && enc, "b2_encode_masks: null argument");
  B2_CHECK(c->cfg.add_mask && c->final_masks, "b2_encode_masks: the context was created without add_mask");
  B2_CHECK(mask_encoder_device(enc) == c->device, "b2_encode_masks: the encoder is bound to another device");
  B2_CHECK(image >= 0 && image < c->cfg.batch, "b2_encode_masks: image out of range");
  if (n < 0 || n > c->cfg.result_per_im) {
    set_error("b2_encode_masks: needs 0 <= n <= result_per_im");
    return kMaskRefused;
  }
  B2_CUDA(cudaSetDevice(c->device));
  const float* masks = c->final_masks + static_cast<size_t>(image) * c->cfg.result_per_im * 784;
  return mask_encode(enc, boxes_host, masks, 1, n, 28, 28, im_h, im_w, offsets_host, bytes_host, capacity, c->stream,
                     "b2_encode_masks");
}

// models.py:517-518, main.py --extract_feat / --just_feat.  With frames the backbone-only pass (main.py's just_feat graph
// stops after the FPN): the detection results and every stage past the FPN still hold an earlier pass's values.
int b2_fpn_feature(b2_ctx* c, const void* frames_host, float* feat_host) {
  B2_CHECK(c && feat_host, "b2_fpn_feature: null argument");
  B2_CUDA(cudaSetDevice(c->device));
  B2_CHECK(c->weights_loaded, "b2_fpn_feature: weights not loaded");
  if (frames_host) {
    B2_CUDA(cudaMemcpyAsync(c->img, frames_host, c->img_bytes, cudaMemcpyHostToDevice, c->stream));
    if (c->cfg.use_cuda_graph) {
      if (!c->feat_graph && capture_graph(c->stream, [c] { return enqueue_feature(c); }, &c->feat_graph)) return -1;
      B2_CUDA(cudaGraphLaunch(c->feat_graph, c->stream));
    } else if (enqueue_feature(c)) {
      return -1;
    }
  } else if (fpn_feature_launch(c)) {
    return -1;
  }
  const size_t bytes = sizeof(float) * c->cfg.batch * 49 * c->cfg.fpn_num_channel;
  B2_CUDA(cudaMemcpyAsync(feat_host, c->fpn_feat, bytes, cudaMemcpyDeviceToHost, c->stream));
  return sync_range(c);
}

// proposal_boxes / proposal_scores of the last pass (models.py:550-558, 2490-2521), as the merge kernel left them.
int b2_get_proposals(b2_ctx* c, float* boxes, float* scores, int32_t* count) {
  B2_CHECK(c && boxes && scores && count, "b2_get_proposals: null argument");
  B2_CUDA(cudaSetDevice(c->device));
  const size_t n = static_cast<size_t>(c->cfg.batch) * c->cfg.rpn_topk;
  cudaStream_t st = c->stream;
  B2_CUDA(cudaMemcpyAsync(boxes, c->rpn.prop_boxes, sizeof(float) * n * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(scores, c->rpn.prop_scores, sizeof(float) * n, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(count, c->rpn.prop_count, sizeof(int32_t) * c->cfg.batch, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// The use_cpu_nms outputs (models.py:899-916) of image `image` of the last pass: the K proposals' boxes of every class, their
// probabilities and the proposals themselves, laid out on the device and copied once K is known.
int b2_get_all_boxes(b2_ctx* c, int image, float* boxes, float* probs, float* rois, int32_t* k_out) {
  B2_CHECK(c && boxes && probs && rois && k_out, "b2_get_all_boxes: null argument");
  B2_CHECK(image >= 0 && image < c->cfg.batch, "b2_get_all_boxes: image out of range");
  B2_CUDA(cudaSetDevice(c->device));
  const int K = c->cfg.rpn_topk, ncls = c->post.num_class, nc1 = ncls - 1;
  cudaStream_t st = c->stream;
  if (!c->all_boxes) {
    c->all_boxes = c->plan.arena.alloc<float>(static_cast<size_t>(nc1) * K * 4, /*zero=*/false);   // written before read
    c->all_probs = c->plan.arena.alloc<float>(static_cast<size_t>(nc1) * K, /*zero=*/false);
    B2_CHECK(c->all_boxes && c->all_probs, "out of device memory (b2_get_all_boxes)");
  }
  const size_t m = static_cast<size_t>(image) * K;
  all_boxes_kernel<<<(nc1 * K + 255) / 256, 256, 0, st>>>(reinterpret_cast<const float4*>(c->post.dec_boxes) + m * nc1,
                                                          c->post.probs + m * ncls, c->rpn.prop_count + image, K, nc1, ncls,
                                                          reinterpret_cast<float4*>(c->all_boxes), c->all_probs);
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(k_out, c->rpn.prop_count + image, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  const size_t n = static_cast<size_t>(*k_out);
  B2_CHECK(*k_out >= 0 && *k_out <= K, "b2_get_all_boxes: proposal count out of range");
  B2_CUDA(cudaMemcpyAsync(boxes, c->all_boxes, sizeof(float) * nc1 * n * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(probs, c->all_probs, sizeof(float) * nc1 * n, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(rois, c->rpn.prop_boxes + m * 4, sizeof(float) * n * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int b2_get_small_objects(b2_ctx* c, float* boxes, float* probs, int32_t* labels, int32_t* count, int32_t* class_counts,
                         int32_t* status) {
  B2_CHECK(c && boxes && probs && labels && count && class_counts && status, "b2_get_small_objects: null argument");
  B2_CHECK(c->ext4.use_small_object_head, "b2_get_small_objects: the context was created without use_small_object_head");
  B2_CUDA(cudaSetDevice(c->device));
  const int R = c->cfg.result_per_im, C = c->so.C;
  cudaStream_t st = c->stream;
  B2_CUDA(cudaMemcpyAsync(boxes, c->so_fin.final_boxes, sizeof(float) * R * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(probs, c->so_fin.final_probs, sizeof(float) * R, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(labels, c->so_fin.final_labels, sizeof(int32_t) * R, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(count, c->so_fin.final_count, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(class_counts, c->so.sel_count, sizeof(int32_t) * C, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(status, c->so.status, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int b2_stage_shape(b2_ctx* c, const char* name, int64_t shape[4], int32_t* dtype) {
  B2_CHECK(c && name && shape, "b2_stage_shape: null argument");
  const Stage* s = c->plan.stages.find(name);
  if (!s) return -1;
  for (int i = 0; i < 4; ++i) shape[i] = s->shape[i];
  if (dtype) *dtype = s->kind == Stage::kI32 ? 1 : 0;
  return 0;
}

int b2_get_stage(b2_ctx* c, const char* name, void* dst, int64_t capacity) {
  B2_CHECK(c && name && dst, "b2_get_stage: null argument");
  B2_CUDA(cudaSetDevice(c->device));
  const Stage* s = c->plan.stages.find(name);
  if (!s) return -1;
  B2_CHECK(capacity >= s->numel() * 4, "b2_get_stage: buffer too small");
  return stage_read(*s, c->stream, dst);
}

int b2_set_stage(b2_ctx* c, const char* name, const void* src, int64_t bytes) {
  B2_CHECK(c && name && src, "b2_set_stage: null argument");
  B2_CUDA(cudaSetDevice(c->device));
  if (strcmp(name, "image") == 0) {
    B2_CHECK(bytes == static_cast<int64_t>(c->img_bytes), "b2_set_stage(image): size mismatch");
    B2_CUDA(cudaMemcpyAsync(c->img, src, bytes, cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
    return 0;
  }
  const Stage* s = c->plan.stages.find(name);
  if (!s) return -1;
  B2_CHECK(bytes == s->numel() * 4, "b2_set_stage: size mismatch");
  return stage_write(*s, c->stream, src);
}

}  // extern "C"
