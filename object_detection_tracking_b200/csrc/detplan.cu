// The detector plan's builders and weight loader (see detplan.h).
#include <float.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <cmath>

#include "detplan.h"

namespace b2 {

namespace {

const char* step_kind_name(StepKind kind) {
  switch (kind) {
#define B2_STEP_KIND_NAME(e, v, n) \
  case e:                          \
    return n;
    B2_STEP_KINDS(B2_STEP_KIND_NAME)
#undef B2_STEP_KIND_NAME
  }
  return "";
}

// The operands of layer L over images [b0, ...): each offset by whole images of its own buffer (a view's pixel stride
// and pitch, not the view's extent)
ConvIO images(const ConvLayer& L, int b0) {
  const ConvDesc& d = L.d;
  auto at = [b0](auto* p, int H, int W, int C) { return p ? p + static_cast<size_t>(b0) * H * W * C : p; };
  ConvIO io = L.io;
  io.in_hi = at(io.in_hi, d.in_pitch_H, d.in_pitch_W, d.in_ld);
  io.in_lo = at(io.in_lo, d.in_pitch_H, d.in_pitch_W, d.in_ld);
  io.out_hi = at(io.out_hi, d.out_H, d.out_W, d.ldc);
  io.out_lo = at(io.out_lo, d.out_H, d.out_W, d.ldc);
  io.out_f32 = at(io.out_f32, d.out_H, d.out_W, d.ldc);
  io.res_hi = at(io.res_hi, d.res_H, d.res_W, d.ldr);
  io.res_lo = at(io.res_lo, d.res_H, d.res_W, d.ldr);
  return io;
}

ConvLayer* add_layer(DetPlan& p, int phase, const std::string& name, const Planes& in, ConvDesc d, ConvAffine affine,
                     const Planes& out, const Planes* res, float* out_f32, int ldc_f32, Layout layout,
                     const ConvLayer* shared = nullptr) {
  d.acc_kb = p.acc_kb;
  if (!res) d.res_shift = 0;
  // the CUDA-core kernel runs a grouped conv as the dense conv with block-diagonal weights
  std::unique_ptr<ConvLayer> L = make_conv(p.arena, p.split, name, d, in, out, res, out_f32, ldc_f32, p.conv_impl != 0,
                                           shared ? &shared->w : nullptr);
  L->bn = affine == kBatchNorm ? name + "/bn" : "";
  L->bias = affine == kBias ? name + "/b" : "";
  L->layout = layout;
  L->io.range_flag = p.range_flag;
  ConvLayer* raw = L.get();
  p.layers.push_back(std::move(L));
  if (phase <= 2) p.part_layers.push_back(raw);
  // algorithmic FLOPs (a grouped conv's output reads Cin / groups channels per tap) and HBM bytes (each operand read
  // once -- the weights as packed --, output written once, at the stored precision)
  const ConvDesc& e = raw->d;
  const double esz = p.split ? 4.0 : 2.0;
  const double M = static_cast<double>(e.B) * e.Ho() * e.Wo();
  const double K = static_cast<double>(e.R) * e.S * e.Cin / e.groups;
  const double in_px = static_cast<double>(e.B) * e.in_H * e.in_W;
  const int conv_impl = p.conv_impl;
  const bool split = p.split;
  Step& s = add_batch_step(p, phase, kStepConv,
                           name + " [" + std::to_string(e.in_H) + "x" + std::to_string(e.in_W) + "x" + std::to_string(e.Cin) + " " +
                               std::to_string(e.R) + "x" + std::to_string(e.S) + "/" + std::to_string(e.stride) + " d" +
                               std::to_string(e.dil) + " ->" + std::to_string(e.Cout) + "]",
                           [raw, conv_impl, split](int, int, cudaStream_t st) {
                             if (conv_impl == 0) return conv_tc_launch(raw->plan.get(), st);
                             return conv_simt_launch(raw->d, raw->w, raw->io, split, st);
                           });
  for (size_t h = 0; h < s.parts.size(); ++h)
    s.parts[h] = [raw, h](cudaStream_t st) { return conv_tc_launch(raw->part_plan[h].get(), st); };
  s.flops = 2.0 * M * K * e.Cout;
  s.bytes = in_px * (e.in_ld > 0 && e.in_ld < e.Cin ? e.in_ld : e.Cin) * esz + static_cast<double>(raw->w.K) * e.Cout * esz +
            M * e.Cout * (raw->io.out_f32 ? 4.0 : esz) + (raw->io.res_hi ? M * e.Cout * esz / (e.res_shift ? 4.0 : 1.0) : 0.0);
  return raw;
}

}  // namespace

Step& add_batch_step(DetPlan& p, int phase, StepKind kind, const std::string& name,
                     const std::function<int(int, int, cudaStream_t)>& launch, int launches) {
  const int B = p.batch;
  Step& s = add_step(p.steps, phase, kind, name.empty() ? step_kind_name(kind) : name,
                     [launch, B](cudaStream_t st) { return launch(0, B, st); }, 0, 0, launches);
  if (p.dual && phase <= 2) {
    const int hb = B / p.nsplit;
    for (int h = 0; h < p.nsplit; ++h) s.parts.push_back([launch, h, hb](cudaStream_t st) { return launch(h * hb, hb, st); });
  }
  return s;
}

// TF padding SAME (SURVEY Appendix B): the total (out - 1) * stride + 2 * dil + 1 - n puts its odd element at the
// bottom / right: at stride 2 on the even sizes of the backbone 0 / 1, with dilation 2 then 1 / 2.
void same_pads3(int h, int w, ConvDesc& d) {
  int pad[4];
  for (int k = 0; k < 2; ++k) {
    const int n = k == 0 ? h : w, o = (n + d.stride - 1) / d.stride;
    const int total = std::max((o - 1) * d.stride + 2 * d.dil + 1 - n, 0);
    pad[2 * k] = total / 2;
    pad[2 * k + 1] = total - total / 2;
  }
  d.pad_t = pad[0]; d.pad_b = pad[1]; d.pad_l = pad[2]; d.pad_r = pad[3];
}

ConvLayer* add_conv(DetPlan& p, int phase, const std::string& name, const Planes& in, ConvDesc d, ConvAffine affine,
                    const Planes& out, const Planes* res, Layout layout) {
  return add_layer(p, phase, name, in, d, affine, out, res, nullptr, 0, layout);
}

ConvLayer* add_conv_shared(DetPlan& p, int phase, const std::string& name, const Planes& in, const ConvLayer& src,
                           const Planes& out) {
  if (src.d.R != 1 || src.d.S != 1 || in.C != src.d.Cin) {
    set_error("b2_create: " + name + " does not match " + src.name);
    return nullptr;
  }
  ConvDesc d = conv_desc(1, src.d.Cout);
  d.relu = src.d.relu;
  return add_layer(p, phase, name, in, d, kNoAffine, out, nullptr, nullptr, 0, kShared, &src);
}

ConvLayer* add_conv_f32(DetPlan& p, int phase, const std::string& name, const Planes& in, ConvDesc d, ConvAffine affine,
                        float* out_f32, int ldc, Layout layout) {
  return add_layer(p, phase, name, in, d, affine, Planes(), nullptr, out_f32, ldc, layout);
}

// A statistics step and an apply step, or with per_roi one step that normalises each [7][7][C] sample of the box head on
// chip.  Statistics scratch is allocated here, so capture works.
int add_gn(DetPlan& p, int phase, const std::string& name, const Planes& buf, int view_h, int view_w, int off_h, int off_w,
           const Planes* res, int res_shift, bool relu, bool per_roi) {
  std::unique_ptr<GnOp> G(new GnOp());
  G->name = name;
  GnParams base;
  memset(&base, 0, sizeof(base));
  base.H = view_h; base.W = view_w; base.C = buf.C;
  base.pitch_H = buf.H; base.pitch_W = buf.W; base.ld = buf.C; base.off_h = off_h; base.off_w = off_w;
  if (res) { base.res_H = res->H; base.res_W = res->W; base.res_ld = res->C; base.res_shift = res_shift; }
  base.relu = relu ? 1 : 0;
  base.gamma = p.arena.alloc<float>(buf.C);
  base.beta = p.arena.alloc<float>(buf.C);
  base.range_flag = p.range_flag;
  B2_CHECK(base.gamma && base.beta, "out of device memory (GroupNorm " + name + ")");
  if (!per_roi) {
    base.chunks = gn_chunks(view_h, view_w, buf.C);
    base.partial = p.arena.alloc<float>(static_cast<size_t>(buf.B) * base.chunks * 32 * 3);
    base.stats = p.arena.alloc<float>(static_cast<size_t>(buf.B) * 32 * 2);
    base.counter = p.arena.alloc<unsigned int>(buf.B);
    B2_CHECK(base.partial && base.stats && base.counter, "out of device memory (GroupNorm " + name + " statistics)");
  }
  // the launch over images [b0, b0 + n): planes and per-image scratch offset by b0
  const Planes x = buf;
  const Planes r = res ? *res : Planes();
  auto params = [base, x, r, per_roi](int b0, int n) {
    GnParams q = base;
    const Planes xs = x.images(b0, n), rs = r.images(b0, n);
    q.x_hi = xs.hi; q.x_lo = xs.lo; q.y_hi = xs.hi; q.y_lo = xs.lo;
    q.r_hi = rs.hi; q.r_lo = rs.lo;
    if (!per_roi) {
      q.partial += static_cast<size_t>(b0) * q.chunks * 32 * 3;
      q.stats += static_cast<size_t>(b0) * 32 * 2;
      q.counter += b0;
    }
    q.B = n;
    return q;
  };
  G->p = params(0, buf.B);
  p.gns.push_back(std::move(G));
  // bytes: statistics read the view once; apply / per-ROI read it, write it and read the residual (a quarter of the view's
  // size when it is upsampled)
  const GnParams& g = p.gns.back()->p;
  const double esz = p.split ? 4.0 : 2.0;
  const double n = static_cast<double>(g.B) * g.H * g.W * g.C;
  const double apply_bytes = 2.0 * n * esz + (g.r_hi ? n * esz / (g.res_shift ? 4.0 : 1.0) : 0.0);
  const std::string dims = " [" + std::to_string(g.H) + "x" + std::to_string(g.W) + "x" + std::to_string(g.C);
  const std::string epi = std::string(g.r_hi ? (g.res_shift ? " +up2" : " +res") : "") + (g.relu ? " relu" : "") + "]";
  if (per_roi) {   // the box head's samples are ROIs, not images: always the whole buffer
    add_batch_step(p, phase, kStepGnRoi, name + " per-roi" + dims + epi,
                   [g](int, int, cudaStream_t st) { return gn_roi_launch(g, st); }).bytes = apply_bytes;
  } else {
    add_batch_step(p, phase, kStepGnStats, name + " stats" + dims + "]",
                   [params](int b0, int nb, cudaStream_t st) { return gn_stats_launch(params(b0, nb), st); }).bytes = n * esz;
    add_batch_step(p, phase, kStepGnApply, name + " apply" + dims + epi,
                   [params](int b0, int nb, cudaStream_t st) { return gn_apply_launch(params(b0, nb), st); }).bytes = apply_bytes;
  }
  return 0;
}

// Squeeze-excite of the bottleneck `name` (nn.py:506-519) then relu(buf * gate + res) in place (nn.py:520-521, 586-587):
// a squeeze step (per-image channel sums), an excite step (fc1 + ReLU, fc2 + sigmoid -> gate [B][C]) and an apply step
// through GroupNorm's apply path.  Every image has its own scratch, so the per-part launches of the forked phases never
// share a buffer and an image's gate does not depend on its batch.
int add_se(DetPlan& p, int phase, const std::string& name, const Planes& buf, const Planes* res) {
  std::unique_ptr<SeOp> S(new SeOp());
  S->name = name;
  S->C = buf.C;
  S->nr = buf.C / 16;                                 // ch_out // 4 with C = 4 * ch_out
  const int B = buf.B, C = S->C, nr = S->nr, HW = buf.H * buf.W, nch = se_chunks(HW);
  B2_CHECK(nr >= 1 && nr <= se_max_nr(), "b2_create: squeeze-excite width out of range (" + name + ")");
  S->w1 = p.arena.alloc<float>(static_cast<size_t>(C) * nr);
  S->b1 = p.arena.alloc<float>(nr);
  S->w2 = p.arena.alloc<float>(static_cast<size_t>(nr) * C);
  S->b2 = p.arena.alloc<float>(C);
  float* partial = p.arena.alloc<float>(static_cast<size_t>(B) * nch * C);
  float* r_part = p.arena.alloc<float>(static_cast<size_t>(B) * se_fc1_parts() * se_max_nr());
  float* gate = p.arena.alloc<float>(static_cast<size_t>(B) * C);
  B2_CHECK(S->w1 && S->b1 && S->w2 && S->b2 && partial && r_part && gate, "out of device memory (squeeze-excite " + name + ")");
  S->gate = gate;
  const Planes x = buf, r = res ? *res : Planes();
  GnParams base;
  memset(&base, 0, sizeof(base));
  base.H = buf.H; base.W = buf.W; base.C = C;
  base.pitch_H = buf.H; base.pitch_W = buf.W; base.ld = C;
  base.res_H = r.H; base.res_W = r.W; base.res_ld = r.C;
  base.relu = 1;
  base.chunks = gn_chunks(buf.H, buf.W, C);
  base.range_flag = p.range_flag;
  const SeOp* se = S.get();
  p.ses.push_back(std::move(S));
  const double esz = p.split ? 4.0 : 2.0;
  const double n = static_cast<double>(B) * HW * C;
  const std::string dims = " [" + std::to_string(buf.H) + "x" + std::to_string(buf.W) + "x" + std::to_string(C);
  add_batch_step(p, phase, kStepSeSqueeze, name + "/se squeeze" + dims + "]", [x, partial, nch, C](int b0, int nb, cudaStream_t st) {
    const Planes xs = x.images(b0, nb);
    return se_squeeze_launch(xs.hi, xs.lo, nb, xs.H * xs.W, C, partial + static_cast<size_t>(b0) * nch * C, st);
  }).bytes = n * esz;
  p.steps.back().flops = n;
  const size_t rp_img = static_cast<size_t>(se_fc1_parts()) * se_max_nr();
  add_batch_step(p, phase, kStepSeExcite, name + "/se excite [" + std::to_string(C) + "->" + std::to_string(nr) + "->" +
                                             std::to_string(C) + "]",
                 [se, partial, r_part, gate, nch, HW, rp_img](int b0, int nb, cudaStream_t st) {
                   return se_excite_launch(partial + static_cast<size_t>(b0) * nch * se->C, nb, HW, se->C, se->C, se->nr,
                                           r_part + b0 * rp_img, se->w1, se->b1, se->w2, se->b2, 1,
                                           gate + static_cast<size_t>(b0) * se->C, nullptr, 0, nullptr, nullptr, st);
                 }, 2).bytes = B * (static_cast<double>(nch) * C + 2.0 * C * nr + C) * 4.0;
  p.steps.back().flops = B * (static_cast<double>(nch) * C + 4.0 * C * nr);
  add_batch_step(p, phase, kStepSeApply, name + "/se apply" + dims + (res ? " +res" : "") + " relu]",
                 [base, x, r, gate](int b0, int nb, cudaStream_t st) {
    GnParams q = base;
    const Planes xs = x.images(b0, nb), rs = r.images(b0, nb);
    q.x_hi = xs.hi; q.x_lo = xs.lo; q.y_hi = xs.hi; q.y_lo = xs.lo;
    q.r_hi = rs.hi; q.r_lo = rs.lo;
    q.gate = gate + static_cast<size_t>(b0) * q.C;
    q.B = nb;
    return se_apply_launch(q, st);
  }).bytes = 3.0 * n * esz;
  p.steps.back().flops = 3.0 * n;
  return 0;
}

// The relation module `name` (relation_network nn.py:115-190), out = h + output_linear(P . h) (models.py:1044-1054: the
// module's output plus its own input).  Steps:
//   query_key          one N = 2D layer (query_linear | key_linear), fp32 output
//   attend             per image: V^T into the image's P.V weights, then geometry + logits + masked softmax -> P
//   attention_value    per image, one layer of 16K rows: P (rows i * 16 + g) times V^T, landing as the [K][16D] flatten
//   output_linear      dense 16D -> D over the flatten, h added in the epilogue, no ReLU
// An image's ROIs attend to its own proposals only (DESIGN 4, Relation head).
int add_relation(DetPlan& p, const std::string& name, int B, int K, int D, const float* boxes, const int* count,
                 const Planes& h, const Planes& out) {
  const int M = B * K;
  const int Kp = (K + 63) / 64 * 64, Mpad = (M + 127) / 128 * 128, G = kRelGroups;
  if (!p.rel_qk) {
    p.rel_qk = p.arena.alloc<float>(static_cast<size_t>(Mpad) * 2 * D);
    B2_CHECK(p.rel_qk && p.alloc_planes(p.rel_p, B, 1, G * K, Kp) && p.alloc_planes(p.rel_o, 1, 1, Mpad, G * D),
             "out of device memory (relation module scratch)");
  }
  std::unique_ptr<RelOp> R(new RelOp());
  R->name = name;
  R->geo = p.arena.alloc<float>(kRelGeoWeights);
  __half** vt = p.arena.alloc<__half*>(2 * B);
  B2_CHECK(R->geo && vt, "out of device memory (relation module " + name + ")");
  add_conv_f32(p, 5, name + "/query_key", h, conv_desc(1, 2 * D), kNoAffine, p.rel_qk, 2 * D, kRelQK);
  RelationParams rp;
  memset(&rp, 0, sizeof(rp));
  rp.boxes = boxes; rp.count = count;
  rp.qk = p.rel_qk; rp.ldqk = 2 * D; rp.D = D; rp.K = K; rp.Kp = Kp;
  rp.rows = relation_rows_per_block(Kp, D);
  rp.geo = R->geo;
  rp.h_hi = h.hi; rp.h_lo = h.lo;
  rp.p_hi = p.rel_p.hi; rp.p_lo = p.rel_p.lo;
  rp.vt_hi = vt; rp.vt_lo = p.split ? vt + B : nullptr;
  p.rels.push_back(std::move(R));
  const double esz = p.split ? 4.0 : 2.0;
  Step& s = add_batch_step(p, 5, kStepRelationAttend, name + "/attend [" + std::to_string(K) + "x" + std::to_string(K) + "x" +
                                                          std::to_string(G) + "]",
                           [rp](int b0, int nb, cudaStream_t st) { return relation_attend_launch(rp, b0, nb, st); }, 2);
  // at full K: per pair the 4 -> 64 -> 16 geometry net and 16 head dots; query / key read once, V^T and P written once
  s.flops = 2.0 * B * K * K * (4.0 * kRelGeoDim + kRelGeoDim * G + D);
  s.bytes = B * (static_cast<double>(K) * 2 * D * 4 + 2.0 * D * Kp * esz + static_cast<double>(G) * K * Kp * esz);
  std::vector<__half*> tab(2 * B, nullptr);
  for (int b = 0; b < B; ++b) {
    Planes o = p.rel_o;   // image b's 16K rows of D: rows b*K .. b*K + K - 1 of the [Mpad][16D] operand
    const size_t off = static_cast<size_t>(b) * G * K * D;
    o.W = G * K; o.C = D;
    o.hi += off;
    if (o.lo) o.lo += off;
    ConvLayer* L = add_conv(p, 5, name + "/attention_value [image " + std::to_string(b) + "]", p.rel_p.images(b, 1),
                            conv_desc(1, D), kNoAffine, o, nullptr, kRuntime);
    tab[b] = L->w.w_hi;
    tab[B + b] = L->w.w_lo;
  }
  B2_CUDA(cudaMemcpy(vt, tab.data(), tab.size() * sizeof(__half*), cudaMemcpyHostToDevice));
  Planes o = p.rel_o;
  o.W = M;
  add_conv(p, 5, name + "/output_linear", o, conv_desc(1, D), kNoAffine, out, &h, kDense);
  return 0;
}

// person_object_relation (nn.py:194-270): the relation module's steps with the query rows of the C blocks attending to
// the Tp key (person) rows, the value being the key rows themselves.  Steps:
//   query_key          one N = 2D layer over all rows (query_linear | key_linear), fp32 output
//   so_attend          V^T of the key rows into the P.V weights, then geometry + logits + softmax over the key rows -> P
//   attention_value    one layer of 16 C Rq rows: P (rows q * 16 + g) times V^T, landing as the [C Rq][16D] flatten
//   output_linear      dense 16D -> D over the flatten, the query rows added in the epilogue
int add_so_association(DetPlan& p, int phase, const std::string& scope, int C, int Rq, int Tp, const float* boxes,
                       const int* kq, const int* nref, const Planes& rows, const Planes& out) {
  const int D = rows.C, Mq = C * Rq, M = Mq + Tp, G = kRelGroups;
  const int Tpp = (Tp + 63) / 64 * 64, Mpad = (M + 127) / 128 * 128, Mqpad = (Mq + 127) / 128 * 128;
  B2_CHECK(D % 64 == 0 && rows.W == M && out.W == Mq && out.C == D, "b2_create: person_object_relation rows do not match");
  std::unique_ptr<RelOp> R(new RelOp());
  R->name = scope;
  R->geo = p.arena.alloc<float>(kRelGeoWeights);
  float* qk = p.arena.alloc<float>(static_cast<size_t>(Mpad) * 2 * D);
  Planes pp, o;
  B2_CHECK(R->geo && qk && p.alloc_rows(pp, Mq * G, Tpp) && p.alloc_planes(o, 1, 1, Mqpad, G * D),
           "out of device memory (person_object_relation)");
  add_conv_f32(p, phase, scope + "/query_key", rows, conv_desc(1, 2 * D), kNoAffine, qk, 2 * D, kRelQK);
  Planes ov = o;   // the P.V output: 16 rows of D per query row
  ov.W = Mq * G; ov.C = D;
  ConvLayer* pv = add_conv(p, phase, scope + "/attention_value", pp, conv_desc(1, D), kNoAffine, ov, nullptr, kRuntime);
  SoAttendParams ap;
  memset(&ap, 0, sizeof(ap));
  ap.boxes = boxes; ap.kq = kq; ap.nref = nref;
  ap.qk = qk; ap.ldqk = 2 * D; ap.D = D; ap.C = C; ap.Rq = Rq; ap.Tp = Tp; ap.Tpp = Tpp;
  ap.rows = relation_rows_per_block(Tpp, D);
  ap.geo = R->geo;
  const size_t kv = static_cast<size_t>(Mq) * D;
  ap.v_hi = rows.hi + kv; ap.v_lo = rows.lo ? rows.lo + kv : nullptr;
  ap.p_hi = pp.hi; ap.p_lo = pp.lo;
  ap.vt_hi = pv->w.w_hi; ap.vt_lo = pv->w.w_lo;
  p.rels.push_back(std::move(R));
  // the P.V layer was appended before the attend step it depends on: move the attend step in front of it
  Step& s = add_batch_step(p, phase, kStepSoAttend, scope + "/attend [" + std::to_string(Mq) + "x" + std::to_string(Tp) + "x" +
                                                       std::to_string(G) + "]",
                           [ap](int, int, cudaStream_t st) { return so_attend_launch(ap, st); }, 2);
  s.flops = 2.0 * Mq * Tp * (4.0 * kRelGeoDim + kRelGeoDim * G + D);
  s.bytes = static_cast<double>(M) * 2 * D * 4 + (2.0 * D * Tpp + static_cast<double>(G) * Mq * Tpp) * (p.split ? 4.0 : 2.0);
  std::rotate(p.steps.end() - 2, p.steps.end() - 1, p.steps.end());
  o.W = Mq;
  Planes hq = rows;
  hq.W = Mq;
  add_conv(p, phase, scope + "/output_linear", o, conv_desc(1, D), kNoAffine, out, &hq, kDense);
  return 0;
}

// The attention branch of fastrcnn_2fc_head (models.py:1064-1089).  Steps:
//   att_pool    the sum over the 49 bins of each ROI's raw ROIAlign features (att_head.cu: why the 3x3 "attention" conv and
//               its length-1 softmax reduce to that sum)
//   att_trans   dense C -> D + bias + ReLU (a plain [C, D] kernel over the channel vector)
//   att_sum     out = att * 1 + hidden through the squeeze-excite apply path with a [1][D] gate of ones and no ReLU: in
//               fp32 exactly relu(att_trans) + hidden, the reference's order (ReLU before the sum), which conv_tc's
//               epilogue (bias, residual, activation) does not have
// Each row depends on its own ROI only, so a batch's rows are those of its images alone.
int add_att_head(DetPlan& p, const Planes& roi, int C, const Planes& hidden, const Planes& pooled, const Planes& att,
                 const Planes& out) {
  const int M = hidden.W, D = hidden.C;
  B2_CHECK(D >= 64 && D <= 2048 && (D & (D - 1)) == 0,
           "b2_create: use_att_frcnn_head needs fc_head_dim a power of two from 64 to 2048");
  B2_CHECK(pooled.W == M && pooled.C == C && att.W == M && att.C == D && out.W == M && out.C == D,
           "b2_create: attention head rows do not match the box head");
  float* ones = p.arena.alloc<float>(D);
  B2_CHECK(ones, "out of device memory (attention head)");
  const std::vector<float> h_ones(D, 1.f);
  B2_CUDA(cudaMemcpy(ones, h_ones.data(), D * sizeof(float), cudaMemcpyHostToDevice));
  p.att_channels = C;
  const double esz = p.split ? 4.0 : 2.0;
  const std::string rows = " [" + std::to_string(M) + "x";
  Step& sp = add_batch_step(p, 5, kStepAttPool, "fastrcnn/att_pool" + rows + "49x" + std::to_string(C) + "]",
                            [roi, M, C, pooled, flag = p.range_flag](int, int, cudaStream_t st) {
                              return att_pool_launch(roi.hi, roi.lo, M, C, pooled.hi, pooled.lo, flag, st);
                            });
  sp.bytes = static_cast<double>(M) * 49 * C * esz + static_cast<double>(M) * C * esz;
  sp.flops = static_cast<double>(M) * 48 * C;
  ConvDesc d = conv_desc(1, D);
  d.relu = 1;
  add_conv(p, 5, "fastrcnn/att_trans", pooled, d, kBias, att, nullptr, kDense);
  GnParams q;
  memset(&q, 0, sizeof(q));
  q.x_hi = att.hi; q.x_lo = att.lo; q.y_hi = out.hi; q.y_lo = out.lo;
  q.r_hi = hidden.hi; q.r_lo = hidden.lo;
  q.B = 1; q.H = 1; q.W = M; q.C = D;
  q.pitch_H = 1; q.pitch_W = M; q.ld = D;
  q.res_H = 1; q.res_W = M; q.res_ld = D;
  q.gate = ones;
  q.chunks = gn_chunks(1, M, D);
  q.range_flag = p.range_flag;
  Step& ss = add_batch_step(p, 5, kStepAttSum, "fastrcnn/att_sum" + rows + std::to_string(D) + " +res]",
                            [q](int, int, cudaStream_t st) { return se_apply_launch(q, st); });
  ss.bytes = 3.0 * M * D * esz;
  ss.flops = static_cast<double>(M) * D;
  p.stages.planes("att_pool", pooled);
  p.stages.planes("att_trans", att);
  p.stages.planes("att_sum", out);
  return 0;
}

// The deformable conv2 (nn.py:470-486, deformable_conv2d nn.py:1642-1712).  Steps:
//   conv2_offset   the offsets, fp32 [B][Ho][Wo][kDeformOffsetLd]: the reference's 3x3 SAME stride-1 conv (bias, no norm,
//                  no activation) is read at the even centres only, so it runs as a 3x3 stride-2 conv with pad 1 top / left
//                  and 2 * Ho - H bottom (2 * Wo - W right): the same value at each centre, a quarter of the work
//   conv2_sample   the bilinear sampler (deform.cu) -> the operand [B][Ho][Wo][9][C]
//   conv2          a 1x1 conv with K = 9 * C over the operand: the [3,3,C,Cout] kernel packed as a 3x3 conv ([Cout][3][3][C])
//                  lines tap k = ky * 3 + kx up with the operand's tap-major K; no bias, norm or ReLU (activation tf.identity)
// Each image is sampled at its own offsets (DESIGN 4, Deformable conv).
int add_deform(DetPlan& p, const std::string& name, const Planes& in, const Planes& out) {
  const int B = in.B, H = in.H, W = in.W, C = in.C, Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  B2_CHECK(out.H == Ho && out.W == Wo && out.C == C, "b2_create: deformable conv2 output does not match its group");
  float* off = p.arena.alloc<float>(static_cast<size_t>(B) * Ho * Wo * kDeformOffsetLd);
  Planes smp;
  B2_CHECK(off && p.alloc_planes(smp, B, Ho, Wo, 9 * C), "alloc deformable operand");
  ConvDesc od = conv_desc(3, 18);
  od.stride = 2;
  od.pad_t = 1; od.pad_b = 2 * Ho - H; od.pad_l = 1; od.pad_r = 2 * Wo - W;
  add_conv_f32(p, 0, name + "/conv2_offset", in, od, kBias, off, kDeformOffsetLd);
  DeformParams dp;
  dp.in_hi = in.hi; dp.in_lo = in.lo;
  dp.offset = off; dp.ld_off = kDeformOffsetLd;
  dp.H = H; dp.W = W; dp.C = C; dp.Ho = Ho; dp.Wo = Wo;
  dp.out_hi = smp.hi; dp.out_lo = smp.lo;
  const double esz = p.split ? 4.0 : 2.0;
  const double taps = 9.0 * B * Ho * Wo;
  Step& s = add_batch_step(p, 0, kStepDeformSample, name + "/conv2_sample [" + std::to_string(H) + "x" + std::to_string(W) +
                                                        "x" + std::to_string(C) + " ->" + std::to_string(Ho) + "x" +
                                                        std::to_string(Wo) + "x9x" + std::to_string(C) + "]",
                           [dp](int b0, int n, cudaStream_t st) { return deform_sample_launch(dp, b0, n, st); });
  // the input read once (the four corners of every sample are mostly L2 hits), the offsets once, the operand written once;
  // three lerps of three operations per sample
  s.bytes = static_cast<double>(B) * H * W * C * esz + B * static_cast<double>(Ho) * Wo * 18 * 4.0 + taps * C * esz;
  s.flops = 9.0 * taps * C;
  add_conv(p, 0, name + "/conv2", smp, conv_desc(1, C), kNoAffine, out);
  p.stages.raw(name + "/conv2_offset", off, Stage::kF32, B, Ho, Wo, kDeformOffsetLd);
  p.stages.planes(name + "/conv2_sample", smp);
  return 0;
}

// The mask head.  Steps:
//   roialign_mask    ROIAlign 14 (a 28 x 28 crop, 2 x 2 average, models.py:936-937) of the boxes into buf.roi
//   fcn0..fcn3       conv 3x3 SAME + bias + ReLU on the [M][14][14][C] maps (M small images)
//   deconv           Conv2DTranspose 2x2 stride 2 + bias + ReLU: no overlap between taps, so a 1x1 conv onto (tap,
//                    channel) outputs (load_layer's kDeconv packing)
//   conv             the 1x1 class conv commutes with the pixel shuffle: it runs on the (pixel, tap) rows directly,
//                    fp32 output
//   mask_select      the logits of each box's own class, sigmoid, un-shuffled to 28 x 28 (mask_head.cu)
// It keeps the checkpoint's num_class - 1 channels with use_partial_classes too, and mask_select reads channel
// (label - 1) for the partial label, as the reference's gather_nd on the full mask logits does (models.py:954-958).
int add_mask_head(DetPlan& p, RoiAlignParams roi, int num_class, const MaskBufs& buf, const int* labels, float* logits,
                  float* masks) {
  const int M = roi.B * roi.rois_per_image, C = roi.C;
  B2_CHECK(num_class >= 2, "b2_create: add_mask needs at least one foreground class");
  const Planes* io[6] = {&buf.roi, &buf.fcn[0], &buf.fcn[1], &buf.fcn[2], &buf.fcn[3], &buf.up};
  for (int k = 0; k < 6; ++k)
    B2_CHECK(io[k]->B == M && io[k]->H == 14 && io[k]->W == 14 && io[k]->C == (k == 5 ? 4 * C : C),
             "b2_create: mask head buffers do not match its boxes");
  roi.out_hi = buf.roi.hi; roi.out_lo = buf.roi.lo; roi.out_nchw = nullptr; roi.out_res = 14;
  add_batch_step(p, 7, kStepRoialignMask, "", [roi](int, int, cudaStream_t st) { return roialign_launch(roi, st); });
  ConvDesc fcn = conv_desc(3, C);
  pad_all(fcn, 1);
  fcn.relu = 1;
  for (int k = 0; k < 4; ++k)
    add_conv(p, 7, "maskrcnn/fcn" + std::to_string(k), k ? buf.fcn[k - 1] : buf.roi, fcn, kBias, buf.fcn[k]);
  ConvDesc deconv = conv_desc(1, 4 * C);
  deconv.relu = 1;
  add_conv(p, 7, "maskrcnn/deconv", buf.fcn[3], deconv, kBias, buf.up, nullptr, kDeconv);
  const int rows = M * 196 * 4;
  Planes up_rows = buf.up;
  up_rows.B = 1; up_rows.H = 1; up_rows.W = rows; up_rows.C = C;
  const int ld = mask_logits_ld(num_class);
  add_conv_f32(p, 7, "maskrcnn/conv", up_rows, conv_desc(1, num_class - 1), kBias, logits, ld);
  const int B = roi.B, R = roi.rois_per_image;
  const int* count = roi.count;
  add_batch_step(p, 7, kStepMaskSelect, "", [logits, ld, labels, count, B, R, masks](int, int, cudaStream_t st) {
    return mask_select_launch(logits, ld, labels, count, B, R, masks, st);
  });
  return 0;
}

// The basic block (resnet_basicblock nn.py:439-456, resnet_shortcut :551-566, the group's ReLU :586-587) into buf.out
// (feat channels): conv1 3x3 at `stride`, SAME, NormReLU into t1; the shortcut (`x` itself when it already has feat
// channels, else convshortcut + norm into sc); conv2 3x3 stride 1 SAME, norm, + shortcut, ReLU.  With BatchNorm the
// norm, shortcut and ReLU are conv epilogues; with GroupNorm the apply steps carry them.  The block has no dilation,
// deformable or squeeze-excite branch.
int add_basic_block(DetPlan& p, const std::string& name, const Planes& x, int stride, const BlockBufs& buf, bool gn) {
  const Planes &t1 = buf.t1, &sc = buf.sc, &out = buf.out;
  const int feat = out.C;
  const ConvAffine norm = gn ? kNoAffine : kBatchNorm;
  ConvDesc d1 = conv_desc(3, feat);
  d1.stride = stride;
  same_pads3(x.H, x.W, d1);
  d1.relu = !gn;
  ConvLayer* L1 = add_conv(p, 0, name + "/conv1", x, d1, norm, t1);
  B2_CHECK(L1->d.Ho() == t1.H && L1->d.Wo() == t1.W, "b2_create: basic-block conv1 output does not match its group");
  if (gn && add_gn(p, 0, name + "/conv1/gn", t1, t1.H, t1.W, 0, 0, nullptr, 0, true)) return -1;
  const Planes* resid = &x;
  if (x.C != feat) {
    // stride 2: drop the last row / column, 1x1 stride-2 VALID (nn.py:554-559)
    ConvDesc ds = conv_desc(1, feat);
    ds.stride = stride;
    ds.pad_b = ds.pad_r = 1 - stride;
    ConvLayer* S = add_conv(p, 0, name + "/convshortcut", x, ds, norm, sc);
    B2_CHECK(S->d.Ho() == sc.H && S->d.Wo() == sc.W, "b2_create: basic-block shortcut output does not match its group");
    if (gn && add_gn(p, 0, name + "/convshortcut/gn", sc, sc.H, sc.W, 0, 0, nullptr, 0, false)) return -1;
    resid = &sc;
  }
  ConvDesc d2 = conv_desc(3, feat);
  pad_all(d2, 1);
  d2.relu = !gn;
  add_conv(p, 0, name + "/conv2", t1, d2, norm, out, gn ? nullptr : resid);
  if (gn && add_gn(p, 0, name + "/conv2/gn", out, out.H, out.W, 0, 0, resid, 0, true)) return -1;
  return 0;
}

// The bottleneck (resnet_bottleneck nn.py:459-521, resnet_shortcut :551-566, the group's ReLU :586-587) into buf.out
// (4 * ch_out channels): conv1 1x1 into t1, conv2 3x3 into t2, conv3 1x1 into out with the shortcut (`x`, or convshortcut
// into sc).
int add_bottleneck(DetPlan& p, const std::string& name, const Planes& x, int stride, int dil, const BlockBufs& buf, bool gn,
                   bool se, bool rx, bool deform) {
  const Planes &a1 = buf.t1, &a2 = buf.t2, &sc = buf.sc, &out = buf.out;
  const int mid = a1.C, feat4 = out.C;
  const ConvAffine norm = gn ? kNoAffine : kBatchNorm;
  ConvDesc d1 = conv_desc(1, mid);
  d1.relu = !gn;
  add_conv(p, 0, name + "/conv1", x, d1, norm, a1);
  if (gn && add_gn(p, 0, name + "/conv1/gn", a1, a1.H, a1.W, 0, 0, nullptr, 0, true)) return -1;
  if (deform) {
    // use_deformable (nn.py:470-486, 577-581): a stride-2 block among the last 3 of its group
    B2_CHECK(dil == 1, "b2_create: use_deformable cannot be combined with use_dilations: " + name + " pads its deformable "
                       "conv2 output [1, 0] (nn.py:493-497), but that output is ceil(h/2), not the dilated conv's h/2 - 1, "
                       "so the reference's residual sum fails (24x41 against 23x40 at 720x1280)");
    if (add_deform(p, name, a1, a2)) return -1;
  } else if (rx) {
    // 3x3 split=32, padding SAME (nn.py:537-540); nothing follows the conv (no [1,0] pad, no output offset)
    ConvDesc d2 = conv_desc(3, mid);
    d2.stride = stride;
    d2.dil = dil;
    same_pads3(a1.H, a1.W, d2);
    d2.relu = !gn;
    d2.groups = 32;
    ConvLayer* L2 = add_conv(p, 0, name + "/conv2", a1, d2, norm, a2, nullptr, kGrouped);
    B2_CHECK(L2->d.Ho() == a2.H && L2->d.Wo() == a2.W, "b2_create: ResNeXt conv2 output does not match its group");
    if (gn && add_gn(p, 0, name + "/conv2/gn", a2, a2.H, a2.W, 0, 0, nullptr, 0, true)) return -1;
  } else if (stride == 2) {
    // pad [1,0] + 3x3 stride-2 VALID (nn.py:487-492); with dilation the output is padded [1,0] again
    // (nn.py:493-497): written at offset (1,1) of a buffer whose first row/col stay zero.  GroupNorm + ReLU run
    // before that pad (nn.py:490-497): their view is the conv output, so the pad row / column stay out of the
    // statistics and stay 0.
    ConvDesc d2 = conv_desc(3, mid);
    d2.stride = 2;
    d2.dil = dil;
    d2.pad_t = d2.pad_l = 1;
    d2.relu = !gn;
    d2.off_h = d2.off_w = dil != 1 ? 1 : 0;
    ConvLayer* L2 = add_conv(p, 0, name + "/conv2", a1, d2, norm, a2);
    if (gn && add_gn(p, 0, name + "/conv2/gn", a2, L2->d.Ho(), L2->d.Wo(), d2.off_h, d2.off_w, nullptr, 0, true)) return -1;
  } else {
    ConvDesc d2 = conv_desc(3, mid);
    d2.dil = dil;
    pad_all(d2, dil);
    d2.relu = !gn;
    add_conv(p, 0, name + "/conv2", a1, d2, norm, a2);
    if (gn && add_gn(p, 0, name + "/conv2/gn", a2, a2.H, a2.W, 0, 0, nullptr, 0, true)) return -1;
  }
  const Planes* resid = &x;
  if (x.C != feat4) {
    // resnet_shortcut (nn.py:551-566): stride 2 => drop last row/col, 1x1 stride-2 VALID
    ConvDesc ds = conv_desc(1, feat4);
    ds.stride = stride;
    ds.pad_b = ds.pad_r = 1 - stride;
    add_conv(p, 0, name + "/convshortcut", x, ds, norm, sc);
    if (gn && add_gn(p, 0, name + "/convshortcut/gn", sc, sc.H, sc.W, 0, 0, nullptr, 0, false)) return -1;
    resid = &sc;
  }
  // relu(norm(conv3) + shortcut) (nn.py:512-521, 586-587): with BatchNorm in the conv epilogue, with GroupNorm in its
  // apply step; with use_se the norm alone, then the gate, the shortcut and the ReLU in the SE apply step
  const bool epi = !gn && !se;
  ConvDesc d3 = conv_desc(1, feat4);
  d3.relu = epi;
  add_conv(p, 0, name + "/conv3", a2, d3, norm, out, epi ? resid : nullptr);
  if (gn && add_gn(p, 0, name + "/conv3/gn", out, out.H, out.W, 0, 0, se ? nullptr : resid, 0, !se)) return -1;
  if (se && add_se(p, 0, name, out, resid)) return -1;
  return 0;
}

int plan_layers(DetPlan& p, int num_sms) {
  if (p.conv_impl != 0) return 0;
  if (plan_convs(p.layers, p.split, num_sms)) return -1;
  // the forked layers over each part of the batch: operands offset by whole images of their own buffers
  for (ConvLayer* L : p.part_layers) {
    if (!p.dual) break;
    for (int h = 0; h < p.nsplit; ++h) {
      ConvDesc d = L->d;
      d.B = p.batch / p.nsplit;
      L->part_plan.emplace_back(conv_tc_plan_create(d, L->w, images(*L, h * d.B), p.split, num_sms));
      if (!L->part_plan.back()) {
        set_error(std::string("half-batch plan for ") + L->name + ": " + last_error());
        return -1;
      }
    }
  }
  return 0;
}

namespace {

// ---- weight loading -------------------------------------------------------------------------
// geo_emb (dense 4 -> 64, nn.py:125-127) and geo_conv (1x1 conv 64 -> 16, nn.py:133-135) of a relation module
int load_rel(const RelOp* R, const WeightSet& ws, cudaStream_t st) {
  const float* ew = ws.get(R->name + "/geo_emb/W", 4 * kRelGeoDim);
  const float* eb = ws.get(R->name + "/geo_emb/b", kRelGeoDim);
  const float* cw = ws.get(R->name + "/geo_conv/W", kRelGeoDim * kRelGroups);
  const float* cb = ws.get(R->name + "/geo_conv/b", kRelGroups);
  if (!ew || !eb || !cw || !cb) return -1;
  return relation_upload_geo(ew, eb, cw, cb, R->geo, st);
}

// fastrcnn/attention/{W,b} [3,3,C,1], [1] (models.py:1075-1077) are never computed with (att_head.cu); their only use is
// this check, the condition that keeps every logit of finite fp16-plane features (|x| < 65536) finite, and so its
// length-1 softmax exactly 1
int load_att(int C, const WeightSet& ws) {
  const float* w = ws.get("fastrcnn/attention/W", 9 * static_cast<int64_t>(C));
  const float* b = ws.get("fastrcnn/attention/b", 1);
  if (!w || !b) return -1;
  double s = 0.0;
  for (int i = 0; i < 9 * C; ++i) {
    B2_CHECK(std::isfinite(w[i]), "attention head: fastrcnn/attention/W not finite");
    s += fabs(static_cast<double>(w[i]));
  }
  B2_CHECK(std::isfinite(b[0]), "attention head: fastrcnn/attention/b not finite");
  B2_CHECK(65536.0 * s + fabs(static_cast<double>(b[0])) < static_cast<double>(FLT_MAX),
           "attention head: fastrcnn/attention/W too large: 65536 * sum|W| + |b| reaches FLT_MAX, so a logit of finite "
           "features could overflow");
  return 0;
}

int load_layer(const ConvLayer* L, const WeightSet& ws, int num_class, const int* partial_ids, int num_partial,
               cudaStream_t st) {
  if (L->layout == kRuntime || L->layout == kShared) return 0;   // written by the pass itself / another layer's
  const int Cin = L->d.Cin, R = L->d.R, S = L->d.S, Cout = L->d.Cout, K = L->w.K, Cp = L->w.Cout_pad;
  std::vector<float> packed(static_cast<size_t>(Cp) * K, 0.f);
  std::vector<double> scale, shift;
  // BatchNorm inference (nn.py:1771-1774, eps 1e-5)
  if (fold_bn(ws, L->bn, kTensorpackBn, 1e-5, Cout, scale, shift)) return -1;
  std::vector<float> b(Cout, 0.f);   // the layer's bias, when it has one
  bool has_b = !L->bias.empty();
  if (L->layout == kHwio) {
    const float* w = ws.get(L->name + "/W", static_cast<int64_t>(R) * S * Cin * Cout);   // HWIO
    if (!w) return -1;
    for (int t = 0; t < R * S; ++t)
      for (int ci = 0; ci < Cin; ++ci) {
        const float* src = w + (static_cast<size_t>(t) * Cin + ci) * Cout;
        for (int o = 0; o < Cout; ++o)
          packed[static_cast<size_t>(o) * K + static_cast<size_t>(t) * Cin + ci] = static_cast<float>(src[o] * scale[o]);
      }
  } else if (L->layout == kGrouped) {
    // ResNeXt conv2 (split=32): HWIO [R][S][Cin/groups][Cout], output o reading the input channels of its group
    const float* w = ws.get(L->name + "/W", static_cast<int64_t>(R) * S * (Cin / L->d.groups) * Cout);
    if (!w) return -1;
    pack_grouped(w, R * S, Cin, Cout, L->d.groups, scale.data(), K, packed);
  } else if (L->layout == kDeconv) {
    // tf.layers.Conv2DTranspose kernel [kh=2, kw=2, out, in] (nn.py:402-412): output row (dy*2+dx)*out + o of the 1x1 conv
    const int co = Cout / 4;
    const float* w = ws.get(L->name + "/W", static_cast<int64_t>(4) * co * Cin);
    const float* bb = ws.get(L->bias, co);
    if (!w || !bb) return -1;
    for (int t = 0; t < 4; ++t)
      for (int o = 0; o < co; ++o) {
        const float* src = w + (static_cast<size_t>(t) * co + o) * Cin;
        for (int ci = 0; ci < Cin; ++ci) packed[static_cast<size_t>(t * co + o) * K + ci] = src[ci];
        b[t * co + o] = bb[o];
      }
    has_b = false;
  } else if (L->layout == kStem) {
    // stem: reference HWIO [7,7,3,64] re-indexed for the packed operand (stem.cu):
    // W'[o][r][s*16 + ry*6 + sx*3 + c] = W[2r+ry][2s+sx][c][o]   (12 real + 4 zero channels per width tap s)
    const float* w = ws.get(L->name + "/W", 7 * 7 * 3 * 64);
    if (!w) return -1;
    for (int r = 0; r < 4; ++r)
      for (int ch = 0; ch < 64; ++ch) {
        const int s4 = ch / 16, r12 = ch % 16, ry = r12 / 6, sx = (r12 % 6) / 3, cc = r12 % 3;
        const int rr = 2 * r + ry, ss = 2 * s4 + sx;
        if (r12 >= 12 || rr >= 7 || ss >= 7) continue;
        const float* src = w + (static_cast<size_t>(rr * 7 + ss) * 3 + cc) * 64;
        for (int o = 0; o < Cout; ++o)
          packed[static_cast<size_t>(o) * K + static_cast<size_t>(r) * Cin + ch] = static_cast<float>(src[o] * scale[o]);
      }
  } else if (L->layout == kFc6) {
    // fc6 (and the conv head's fc): reference flattens NCHW (index c*49 + y*7 + x, models.py:1056 + nn.py:738-740);
    // our ROI features are [y][x][c], so permute the rows of W [in, out].
    const int C = Cin / 49;
    const float* w = ws.get(L->name + "/W", static_cast<int64_t>(Cin) * Cout);
    if (!w) return -1;
    for (int ch = 0; ch < C; ++ch)
      for (int s = 0; s < 49; ++s) {
        const float* src = w + (static_cast<size_t>(ch) * 49 + s) * Cout;
        const size_t k = static_cast<size_t>(s) * C + ch;
        for (int o = 0; o < Cout; ++o) packed[static_cast<size_t>(o) * K + k] = src[o];
      }
  } else if (L->layout == kRelQK) {
    // relation module query_linear / key_linear (nn.py:146-156): dense D -> D each, no bias, one N = 2D layer
    const std::string scope = L->name.substr(0, L->name.rfind('/'));
    const float* wq = ws.get(scope + "/query_linear/W", static_cast<int64_t>(Cin) * Cin);
    const float* wk = ws.get(scope + "/key_linear/W", static_cast<int64_t>(Cin) * Cin);
    if (!wq || !wk) return -1;
    relation_pack_qk(wq, wk, Cin, packed);
  } else if (L->layout == kSoClass) {
    // the per-class [D, 2] layers of the small-object branch (models.py:682-689): class i's columns at 2i, 2i + 1
    for (int i = 0; i < Cout / 2; ++i) {
      const std::string n = "fastrcnn/small_objects/small_object_classification_c" + std::to_string(i + 1);
      const float* w = ws.get(n + "/W", static_cast<int64_t>(Cin) * 2);
      const float* bb = ws.get(n + "/b", 2);
      if (!w || !bb) return -1;
      for (int o = 0; o < 2; ++o) {
        for (int k = 0; k < Cin; ++k) packed[static_cast<size_t>(2 * i + o) * K + k] = w[static_cast<size_t>(k) * 2 + o];
        b[2 * i + o] = bb[o];
      }
    }
    has_b = false;
  } else if (L->layout == kDense) {
    const float* w = ws.get(L->name + "/W", static_cast<int64_t>(Cin) * Cout);
    if (!w) return -1;
    for (int k = 0; k < Cin; ++k)
      for (int o = 0; o < Cout; ++o) packed[static_cast<size_t>(o) * K + k] = w[static_cast<size_t>(k) * Cout + o];
  } else {
    // two reference layers fused along N: rpn/{class,box} or fastrcnn/outputs/{class,box}.  col0 / col1 hold the
    // checkpoint column of each packed class / box column.  use_partial_classes (models.py:807-828) keeps the class
    // columns [0] + partial_ids and the 4 box columns of each kept class; class 0's box columns stay as a slot the decode
    // never reads, so the packed layout is the full one's for num_partial + 1 classes.  A class-agnostic box output (4
    // columns) is kept whole.
    const bool head = L->layout == kHeadOut, part = head && num_partial > 0;
    const std::string base = head ? "fastrcnn/outputs" : "rpn";
    const int n0 = head ? num_class : 3;                        // checkpoint class columns
    const int p0 = part ? num_partial + 1 : n0;                 // packed class columns
    const int p1 = Cout - p0;                                   // packed box columns
    const bool gather_box = part && p1 != 4;
    const int n1 = gather_box ? 4 * num_class : p1;             // checkpoint box columns
    std::vector<int> col0(p0), col1(p1);
    for (int o = 0; o < p0; ++o) col0[o] = part && o > 0 ? partial_ids[o - 1] : o;
    for (int o = 0; o < p1; ++o) col1[o] = gather_box ? col0[o / 4] * 4 + o % 4 : o;
    const float* w0 = ws.get(base + "/class/W", static_cast<int64_t>(Cin) * n0);
    const float* b0 = ws.get(base + "/class/b", n0);
    const float* w1 = ws.get(base + "/box/W", static_cast<int64_t>(Cin) * n1);
    const float* b1 = ws.get(base + "/box/b", n1);
    if (!w0 || !b0 || !w1 || !b1) return -1;
    for (int k = 0; k < Cin; ++k) {
      for (int o = 0; o < p0; ++o) packed[static_cast<size_t>(o) * K + k] = w0[static_cast<size_t>(k) * n0 + col0[o]];
      for (int o = 0; o < p1; ++o) packed[static_cast<size_t>(p0 + o) * K + k] = w1[static_cast<size_t>(k) * n1 + col1[o]];
    }
    for (int o = 0; o < p0; ++o) b[o] = b0[col0[o]];
    for (int o = 0; o < p1; ++o) b[p0 + o] = b1[col1[o]];
    has_b = false;
  }
  if (has_b) {
    const float* bb = ws.get(L->bias, Cout);
    if (!bb) return -1;
    b.assign(bb, bb + Cout);
  }
  return upload_conv(*L, packed, fold_bias(scale, shift, L->bias.empty() ? nullptr : b.data(), Cout, Cp), st);
}

// group_norm's "<scope>/gamma" and "<scope>/beta" (nn.py:97-102), [C] each
int load_gn(const GnOp* G, const WeightSet& ws, cudaStream_t st) {
  const int C = G->p.C;
  const float* g = ws.get(G->name + "/gamma", C);
  const float* b = ws.get(G->name + "/beta", C);
  if (!g || !b) return -1;
  for (int i = 0; i < C; ++i)
    B2_CHECK(std::isfinite(g[i]) && std::isfinite(b[i]), "GroupNorm " + G->name + ": gamma / beta not finite");
  B2_CUDA(cudaMemcpyAsync(const_cast<float*>(G->p.gamma), g, C * sizeof(float), cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaMemcpyAsync(const_cast<float*>(G->p.beta), b, C * sizeof(float), cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// dense "<block>/fc1" and "<block>/fc2" (nn.py:509-514, dense nn.py:730-774): W [in, out] row-contiguous, b [out]
int load_se(const SeOp* S, const WeightSet& ws, cudaStream_t st) {
  const int C = S->C, nr = S->nr;
  const struct { const char* suffix; int64_t n; float* dst; } parts[] = {
      {"/fc1/W", static_cast<int64_t>(C) * nr, S->w1}, {"/fc1/b", nr, S->b1},
      {"/fc2/W", static_cast<int64_t>(nr) * C, S->w2}, {"/fc2/b", C, S->b2}};
  for (const auto& e : parts) {
    const float* h = ws.get(S->name + e.suffix, e.n);
    if (!h) return -1;
    for (int64_t i = 0; i < e.n; ++i)
      B2_CHECK(std::isfinite(h[i]), "squeeze-excite " + S->name + e.suffix + ": not finite");
    B2_CUDA(cudaMemcpyAsync(e.dst, h, e.n * sizeof(float), cudaMemcpyHostToDevice, st));
  }
  B2_CUDA(cudaStreamSynchronize(st));
  return 0;
}

}  // namespace

int load_weights(const DetPlan& p, const WeightSet& ws, int num_class, cudaStream_t st, const int* partial_ids,
                 int num_partial) {
  // shared RPN weights: packed once, every level's layer gets its own copy of the (small) operand
  for (auto& L : p.layers)
    if (load_layer(L.get(), ws, num_class, partial_ids, num_partial, st)) return -1;
  for (auto& G : p.gns)
    if (load_gn(G.get(), ws, st)) return -1;
  for (auto& S : p.ses)
    if (load_se(S.get(), ws, st)) return -1;
  for (auto& R : p.rels)
    if (load_rel(R.get(), ws, st)) return -1;
  if (p.att_channels > 0 && load_att(p.att_channels, ws)) return -1;
  return 0;
}

}  // namespace b2
