// EfficientDet feature network (BiFPN), class/box nets and post-processing behind the C ABI.
// One b2_effdet = one device = one fixed network input size and batch; the pass is a fixed launch sequence replayed as a
// CUDA graph.  The reference wrapper runs one frame per call (efficientdet_wrapper.py:304-363); a context created with
// batch B runs B independent frames per call, each with the batch-1 semantics and bit-identical to a batch-1 context:
// every kernel takes the image from its grid or its row index, the squeeze-excite gate is folded into one copy of the
// projection weights per image and each image's projection is its own conv layer, and the post-processing keeps one
// slice of scratch and outputs per image.
//
// Reference graph: efficientdet_arch.py build_feature_network (:440-505) / build_bifpn_layer (:594-682) /
// resample_feature_map (:105-200) / class_net (:227-282) / box_net (:285-340), then
// efficientdet_wrapper.py add_metric_fn_inputs (:367-474), anchors.py _generate_detections_tf (:399-487) and the
// wrapper's own-level ROIAlign box feature (:265-301).
//
// Every separable conv = depthwise 3x3 kernel (effdet.cu) + pointwise GEMM on the wgmma conv kernel with bias,
// folded BatchNorm (eps 1e-3) and swish in the epilogue.  The class/box nets share conv weights across levels but
// not BatchNorm statistics, so each level gets its own folded copy of the pointwise weights.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/b200det.h"
#include "engine_core.h"
#include "kernels.h"

using namespace b2;

namespace {

struct EDw {
  std::string wname;      // [3,3,C,1]
  Planes in, out;
  float* w = nullptr;     // [9][Cpad]
};

struct ECombine {
  BifpnCombineParams p;
  std::string wnames[3];  // fast-attention scalars
};

// backbone: depthwise KxK + BN + swish
struct EDwBn {
  std::string wname, bnname;
  DwConvParams p;
  float* w = nullptr;
  float* bias = nullptr;
  int creal = 0;
};

// backbone: squeeze-excite whose gate is folded into the projection conv's weights every frame, one copy per image
struct ESe {
  std::string pre;          // ".../blocks_i/se"
  Planes x;
  int creal = 0, nr = 0;
  float *partial = nullptr, *r_part = nullptr, *gate = nullptr, *w1 = nullptr, *b1 = nullptr, *w2 = nullptr, *b2 = nullptr;
  const ConvLayer* proj = nullptr;   // image 0's projection: its w_master holds the BN-folded weights [Cout_pad][K] fp32
  __half *fold_hi = nullptr, *fold_lo = nullptr;   // [B][Cout_pad][K]: image b's projection layer reads slice b
};

// Step phases (bit i of b2_effdet_run_phases' mask = phase i): the backbone runs only in b2_effdet_detect's graph; the
// feature network + heads, the post-processing and the box feature run in both graphs
enum { kBackbone = 0, kFeatures = 1, kPost = 2, kBoxFeat = 3 };

int pad64(int c) { return (c + 63) / 64 * 64; }
int pad16(int c) { return (c + 15) / 16 * 16; }

// anchor_scale and the aspect ratios arrive as float32, but anchors.py builds the grid in float64 from the decimals the
// configuration writes (1.4, 0.7): the shortest decimal that rounds to the float32 is that value.
double config_double(float f) {
  char buf[32];
  for (int p = 1; p <= 9; ++p) {
    snprintf(buf, sizeof(buf), "%.*g", p, static_cast<double>(f));
    const double d = strtod(buf, nullptr);
    if (static_cast<float>(d) == f) return d;
  }
  return f;
}

}  // namespace

struct b2_effdet {
  Arena arena;                       // first member: freed after everything that refers to it
  b2_effdet_config cfg;
  int device = 0, num_sms = 132;
  bool split = true;
  int F = 0, Fp = 0, nlev = 0, na = 0;
  int fh[8] = {0}, fw[8] = {0};               // feature size per level (index = level)
  cudaStream_t stream = nullptr;
  std::vector<std::unique_ptr<ConvLayer>> convs;
  std::vector<std::unique_ptr<EDw>> dws;
  std::vector<std::unique_ptr<ECombine>> combines;
  std::map<std::string, float*> dw_shared;    // depthwise kernels shared across levels
  std::vector<std::unique_ptr<EDwBn>> dwbns;
  std::vector<std::unique_ptr<ESe>> ses;
  std::vector<Step> steps;           // backbone (when cfg.backbone >= 0), feature network, heads, post-processing
  int phase = kFeatures;             // phase of the steps being added
  std::string bb_name;
  int B = 1;                         // images per call
  float* image = nullptr;            // [B][H][W][3] fp32, pre-processed network input
  uint8_t* frame = nullptr;          // device copy of the caller's BGR frames, back to back (grow-only)
  size_t frame_cap = 0;
  EffnetFrame* frame_table = nullptr;   // [B] where each image's frame lies in `frame`, and its sizes
  Planes stem_cols;
  cudaGraphExec_t graph_full = nullptr;
  StageMap named;
  Planes backbone[3];
  Planes fpn_out[5];
  EffdetPostParams post;
  LevelRoiFeatParams roi;
  float* scale_dev = nullptr;        // [B] image_scale of each image
  float4* out_boxes = nullptr;       // outputs [B][max_out] (out_count [B], out_feat [B][max_out][F])
  float* out_scores = nullptr;
  int *out_classes = nullptr, *out_levels = nullptr, *out_count = nullptr;
  float* out_feat = nullptr;
  cudaGraphExec_t graph = nullptr;
  bool loaded = false;

  Planes planes(int h, int w, int c, int creal) { return arena.planes(B, h, w, c, split, creal); }
  double esz() const { return split ? 4.0 : 2.0; }
};

namespace {

// pointwise conv in -> out (planes) or -> fp32 [H*W][ldc32]; act: 0 none, 2 swish
ConvLayer* add_pw(b2_effdet* c, const std::string& wname, const std::string& biasname, const std::string& bn,
                  const Planes& in, const Planes& out, int cout_real, int act, const Planes* res = nullptr,
                  float* out_f32 = nullptr, int ldc32 = 0) {
  ConvDesc d;
  d.Cout = cout_real; d.relu = act;
  // chunked re-accumulation (conv_tc ACC) on every layer with more than one K-block (acc_kb 0 = the kernel's default
  // chunk).  Round 1 switched it off up to K = 512 for speed; at D7 depth (EfficientNet-b6: 45 blocks, then 8 BiFPN cells
  // and 5-deep heads at 1536^2) the truncation bias of up to 32 tensor-core accumulation steps per layer then compounds
  // to 3e-5 relative on c5 -- six times the rounding noise of a float32 evaluation -- and boxes leave the 1e-3 px bar.
  d.acc_kb = 0;
  std::unique_ptr<ConvLayer> L = make_conv(c->arena, c->split, wname, d, in, out, res, out_f32, ldc32);
  L->bias = biasname; L->bn = bn; L->cin_real = in.creal;
  ConvLayer* raw = L.get();
  c->convs.push_back(std::move(L));
  const ConvDesc& e = raw->d;
  const double M = static_cast<double>(e.B) * e.in_H * e.in_W, esz = c->esz();
  Step& s = add_conv_step(c->steps, c->phase, raw);
  s.name = wname + " [" + std::to_string(e.in_H) + "x" + std::to_string(e.in_W) + "x" + std::to_string(raw->cin_real) +
           "->" + std::to_string(cout_real) + "]";
  s.flops = 2.0 * M * raw->cin_real * cout_real;
  s.bytes = M * e.Cin * esz + static_cast<double>(raw->w.K) * raw->w.Cout_pad * esz +
            M * (raw->io.out_f32 ? raw->w.Cout_pad * 4.0 : e.ldc * esz) + (raw->io.res_hi ? M * e.ldr * esz : 0.0);
  return raw;
}

void add_dw(b2_effdet* c, const std::string& wname, const Planes& in, const Planes& out) {
  std::unique_ptr<EDw> D(new EDw());
  D->wname = wname; D->in = in; D->out = out;
  auto it = c->dw_shared.find(wname);
  if (it == c->dw_shared.end()) {
    D->w = c->arena.alloc<float>(9 * static_cast<size_t>(in.C));
    c->dw_shared[wname] = D->w;
  } else {
    D->w = it->second;
  }
  const EDw* e = D.get();
  add_step(c->steps, c->phase, 1, wname, [e](cudaStream_t st) {
    return dw3x3_plain_launch(e->in.hi, e->in.lo, e->in.B, e->in.H, e->in.W, e->in.C, e->w, e->out.hi, e->out.lo, st);
  }, 2.0 * static_cast<double>(in.elems()) * c->esz(), 18.0 * static_cast<double>(in.B) * in.H * in.W * in.creal);
  c->dws.push_back(std::move(D));
}

void add_combine(b2_effdet* c, std::unique_ptr<ECombine> K) {
  const BifpnCombineParams& p = K->p;
  double in = 0;
  for (int i = 0; i < p.n_in; ++i) in += static_cast<double>(p.in[i].H) * p.in[i].W * p.C;
  const ECombine* k = K.get();
  add_step(c->steps, c->phase, 2,
           "combine x" + std::to_string(p.n_in) + " [" + std::to_string(p.Ho) + "x" + std::to_string(p.Wo) + "]",
           [k](cudaStream_t st) { return bifpn_combine_launch(k->p, st); },
           p.B * (in + static_cast<double>(p.Ho) * p.Wo * p.C) * c->esz());
  c->combines.push_back(std::move(K));
}

int set_input(BifpnInput& bi, const Planes& src, int th, int tw) {
  return bifpn_set_input(bi, src.hi, src.lo, src.H, src.W, th, tw);
}

// resample_feature_map's optional 1x1 conv + BN (at the source resolution), arch.py:131-146
Planes maybe_1x1(b2_effdet* c, const Planes& src, const std::string& name) {
  if (src.creal == c->F) return src;
  Planes t = c->planes(src.H, src.W, c->Fp, c->F);
  add_pw(c, name + "/conv2d/kernel", name + "/conv2d/bias", name + "/bn", src, t, c->F, 0);
  return t;
}

int add_pool(b2_effdet* c, const Planes& src, const Planes& dst) {
  std::unique_ptr<ECombine> K(new ECombine());
  memset(&K->p, 0, sizeof(K->p));
  if (set_input(K->p.in[0], src, dst.H, dst.W)) return -1;
  K->p.n_in = 1; K->p.B = c->B; K->p.Ho = dst.H; K->p.Wo = dst.W; K->p.C = dst.C;
  K->p.weighted = 0; K->p.denom = 1.f; K->p.swish = 0;
  K->p.out_hi = dst.hi; K->p.out_lo = dst.lo;
  add_combine(c, std::move(K));
  return 0;
}


struct BlockSpec { int kernel, stride, expand, cin, cout; };

int round_filters(double filters, double width) {
  filters *= width;
  int nf = static_cast<int>(filters + 4.0) / 8 * 8;      // efficientnet_model.py:137-151, divisor 8
  if (nf < 8) nf = 8;
  if (nf < 0.9 * filters) nf += 8;
  return nf;
}

void same_pad(int n, int k, int s, int* out, int* before) {
  *out = (n + s - 1) / s;
  const int total = (*out - 1) * s + k - n;
  *before = (total > 0 ? total : 0) / 2;
}

// EfficientNet-b{0..7} trunk up to reduction_5 (efficientnet_model.py:504-704); endpoints land in c->backbone[0..2]
int build_backbone(b2_effdet* c) {
  static const double kWidth[8] = {1.0, 1.0, 1.1, 1.2, 1.4, 1.6, 1.8, 2.0};
  static const double kDepth[8] = {1.0, 1.1, 1.2, 1.4, 1.8, 2.2, 2.6, 3.1};
  static const int kStage[7][6] = {{1, 3, 1, 1, 32, 16}, {2, 3, 2, 6, 16, 24}, {2, 5, 2, 6, 24, 40}, {3, 3, 2, 6, 40, 80},
                                   {3, 5, 1, 6, 80, 112}, {4, 5, 2, 6, 112, 192}, {1, 3, 1, 6, 192, 320}};
  const b2_effdet_config& g = c->cfg;
  B2_CHECK(g.backbone >= 0 && g.backbone <= 7, "effdet: backbone must be efficientnet-b0..b7");
  const double width = kWidth[g.backbone], depth = kDepth[g.backbone];
  c->bb_name = "efficientnet-b" + std::to_string(g.backbone);
  std::vector<BlockSpec> blocks;
  for (const auto& st : kStage) {
    const int rep = static_cast<int>(ceil(depth * st[0])), ci = round_filters(st[4], width), co = round_filters(st[5], width);
    blocks.push_back({st[1], st[2], st[3], ci, co});
    for (int r = 1; r < rep; ++r) blocks.push_back({st[1], 1, st[3], co, co});
  }
  c->phase = kBackbone;
  const int H = g.image_h, W = g.image_w;
  c->image = c->arena.alloc<float>(static_cast<size_t>(c->B) * H * W * 3);
  c->frame_table = c->arena.alloc<EffnetFrame>(c->B);
  c->named.raw("image", c->image, Stage::kF32, c->B, H, W, 3);
  // stem: 3x3/2 SAME as a 1x1 conv over im2col-packed pixels (27 live of 64 operand channels)
  int h = 0, w = 0, pt = 0, pl = 0;
  same_pad(H, 3, 2, &h, &pt);
  same_pad(W, 3, 2, &w, &pl);
  c->stem_cols = c->planes(h, w, 64, 27);
  const Planes cols = c->stem_cols;
  add_step(c->steps, c->phase, 5, "stem_im2col", [c, cols, pt, pl](cudaStream_t st) {
    return stem_im2col_launch(c->image, cols.B, c->cfg.image_h, c->cfg.image_w, cols.H, cols.W, pt, pl, cols.hi, cols.lo, st);
  }, static_cast<double>(c->B) * H * W * 3 * 4 + static_cast<double>(cols.elems()) * c->esz());
  const int stem_c = round_filters(32, width);
  Planes x = c->planes(h, w, pad64(stem_c), stem_c);
  add_pw(c, c->bb_name + "/stem/conv2d/kernel", "", c->bb_name + "/stem/tpu_batch_normalization", c->stem_cols, x, stem_c, 2);
  c->named.planes("stem", x);
  int reduction = 0;   // reduction_k closes when the next block strides or at the last block (Model.call :644-668)
  for (size_t i = 0; i < blocks.size(); ++i) {
    const BlockSpec& b = blocks[i];
    const std::string pre = c->bb_name + "/blocks_" + std::to_string(i);
    B2_CHECK(x.creal == b.cin, "effdet backbone: channel bookkeeping mismatch");
    const int mid = b.cin * b.expand;
    Planes e = x;
    std::string proj = "conv2d";
    if (b.expand != 1) {
      e = c->planes(x.H, x.W, pad64(mid), mid);
      add_pw(c, pre + "/conv2d/kernel", "", pre + "/tpu_batch_normalization", x, e, mid, 2);
      proj = "conv2d_1";
    }
    std::unique_ptr<EDwBn> D(new EDwBn());
    int ho = 0, wo = 0, dpt = 0, dpl = 0;
    same_pad(e.H, b.kernel, b.stride, &ho, &dpt);
    same_pad(e.W, b.kernel, b.stride, &wo, &dpl);
    Planes d = c->planes(ho, wo, e.C, mid);
    D->wname = pre + "/depthwise_conv2d/depthwise_kernel"; D->bnname = pre + "/tpu_batch_normalization_1"; D->creal = mid;
    D->w = c->arena.alloc<float>(static_cast<size_t>(b.kernel) * b.kernel * e.C);
    D->bias = c->arena.alloc<float>(e.C);
    D->p = DwConvParams{e.hi, e.lo, c->B, e.H, e.W, e.C, b.kernel, b.stride, dpt, dpl, ho, wo, D->w, D->bias, d.hi, d.lo};
    const DwConvParams& dp = D->p;
    add_step(c->steps, c->phase, 3,
             D->wname + " [" + std::to_string(dp.H) + "x" + std::to_string(dp.W) + "x" + std::to_string(mid) + " k" +
                 std::to_string(dp.K) + "/" + std::to_string(dp.stride) + "]",
             [dp](cudaStream_t st) { return dwconv_bn_swish_launch(dp, st); },
             dp.B * (static_cast<double>(dp.H) * dp.W + static_cast<double>(dp.Ho) * dp.Wo) * dp.C * c->esz(),
             2.0 * dp.K * dp.K * dp.B * static_cast<double>(dp.Ho) * dp.Wo * mid);
    c->dwbns.push_back(std::move(D));
    // squeeze-excite (se_ratio 0.25 of the block's input filters)
    std::unique_ptr<ESe> S(new ESe());
    S->pre = pre + "/se"; S->x = d; S->creal = mid; S->nr = b.cin / 4 > 1 ? b.cin / 4 : 1;
    S->partial = c->arena.alloc<float>(static_cast<size_t>(c->B) * se_chunks(ho * wo) * d.C);
    S->gate = c->arena.alloc<float>(static_cast<size_t>(c->B) * d.C);
    S->r_part = c->arena.alloc<float>(static_cast<size_t>(c->B) * se_fc1_parts() * se_max_nr());
    S->w1 = c->arena.alloc<float>(static_cast<size_t>(mid) * S->nr); S->b1 = c->arena.alloc<float>(S->nr);
    S->w2 = c->arena.alloc<float>(static_cast<size_t>(S->nr) * mid); S->b2 = c->arena.alloc<float>(mid);
    const ESe* se = S.get();
    add_step(c->steps, c->phase, 4, S->pre, [se](cudaStream_t st) {   // pool + fc1 + fc2 / gate / weight rescale
      const ConvLayer* P = se->proj;
      return se_gate_launch(se->x.hi, se->x.lo, se->x.B, se->x.H * se->x.W, se->x.C, se->creal, se->nr, se->partial,
                            se->r_part, se->w1, se->b1, se->w2, se->b2, se->gate, P->w_master, P->w.Cout_pad, se->fold_hi,
                            se->fold_lo, st);
    }, 0.0, 0.0, 3);
    const size_t se_idx = c->steps.size() - 1;
    c->ses.push_back(std::move(S));
    // projection (+ identity skip when the block keeps shape, efficientnet_model.py:381-390): one layer per image, on its
    // slice of the depthwise output and skip, with its image's folded weights
    Planes y = c->planes(ho, wo, pad64(b.cout), b.cout);
    const bool skip = b.stride == 1 && b.cin == b.cout;
    std::vector<ConvLayer*> P(c->B);
    for (int im = 0; im < c->B; ++im) {
      const Planes xi = x.images(im, 1);
      P[im] = add_pw(c, pre + "/" + proj + "/kernel", "", pre + "/tpu_batch_normalization_2", d.images(im, 1),
                     y.images(im, 1), b.cout, 0, skip ? &xi : nullptr);
      if (c->B > 1) c->steps.back().name += " image " + std::to_string(im);
    }
    const size_t wsz = static_cast<size_t>(P[0]->w.Cout_pad) * P[0]->w.K;
    P[0]->w_master = c->arena.alloc<float>(wsz);
    ESe& se_b = *c->ses.back();
    se_b.proj = P[0];
    if (c->B == 1) {
      se_b.fold_hi = P[0]->w.w_hi; se_b.fold_lo = P[0]->w.w_lo;
    } else {
      se_b.fold_hi = c->arena.alloc<__half>(c->B * wsz);
      se_b.fold_lo = c->split ? c->arena.alloc<__half>(c->B * wsz) : nullptr;
      for (int im = 0; im < c->B; ++im) {
        P[im]->w.w_hi = se_b.fold_hi ? se_b.fold_hi + im * wsz : nullptr;
        P[im]->w.w_lo = se_b.fold_lo ? se_b.fold_lo + im * wsz : nullptr;
      }
    }
    c->steps[se_idx].bytes = static_cast<double>(d.elems()) * c->esz() + (1.0 + c->B) * wsz * 4.0;
    x = y;
    c->named.planes("block_" + std::to_string(i), x);
    if (i + 1 == blocks.size() || blocks[i + 1].stride > 1) {
      const int lvl = ++reduction;
      if (lvl >= 3 && lvl <= 5) {
        B2_CHECK(x.creal == g.backbone_channels[lvl - 3], "effdet: backbone_channels do not match the backbone's endpoints");
        B2_CHECK(x.H == c->fh[lvl] && x.W == c->fw[lvl], "effdet: backbone endpoint size mismatch");
        c->backbone[lvl - 3] = x;
      }
    }
  }
  c->phase = kFeatures;
  return 0;
}

int build(b2_effdet* c) {
  const b2_effdet_config& g = c->cfg;
  B2_CHECK(g.min_level == 3 && g.max_level == 7, "effdet: levels 3..7 only (the reference's configuration)");
  B2_CHECK(g.image_h % 128 == 0 && g.image_w % 128 == 0, "effdet: network input size must be divisible by 128");
  c->F = g.fpn_num_filters; c->Fp = pad64(c->F); c->nlev = 5;
  c->na = g.num_scales * g.num_aspects;
  B2_CHECK(c->na >= 1 && c->na <= 9, "effdet: at most 9 anchors per cell");
  {
    int h = g.image_h, w = g.image_w;
    for (int l = 1; l <= 7; ++l) {
      h = (h - 1) / 2 + 1; w = (w - 1) / 2 + 1;
      c->fh[l] = h; c->fw[l] = w;
    }
  }
  std::vector<Planes> feats;
  if (g.backbone >= 0 && build_backbone(c)) return -1;
  for (int i = 0; i < 3; ++i) {
    const int cr = g.backbone_channels[i];
    if (g.backbone < 0) c->backbone[i] = c->planes(c->fh[3 + i], c->fw[3 + i], pad64(cr), cr);
    feats.push_back(c->backbone[i]);
    c->named.planes("c" + std::to_string(3 + i), c->backbone[i]);
  }
  // P6, P7 (arch.py:464-480): resample_p6 = [conv1x1 + BN] + max-pool, resample_p7 = max-pool
  for (int level = 6; level <= 7; ++level) {
    Planes src = maybe_1x1(c, feats.back(), "resample_p" + std::to_string(level));
    Planes dst = c->planes(c->fh[level], c->fw[level], c->Fp, c->F);
    if (add_pool(c, src, dst)) return -1;
    feats.push_back(dst);
    c->named.planes("p" + std::to_string(level) + "_in", dst);
  }
  static const int node_level[8] = {6, 5, 4, 3, 4, 5, 6, 7};
  static const int node_in[8][3] = {{3, 4, -1}, {2, 5, -1}, {1, 6, -1}, {0, 7, -1}, {1, 7, 8}, {2, 6, 9}, {3, 5, 10}, {4, 11, -1}};
  for (int rep = 0; rep < g.fpn_cell_repeats; ++rep) {
    for (int i = 0; i < 8; ++i) {
      const int lvl = node_level[i], th = c->fh[lvl], tw = c->fw[lvl];
      const std::string pre = "fpn_cells/cell_" + std::to_string(rep) + "/fnode" + std::to_string(i);
      const int nfeats = static_cast<int>(feats.size());
      std::unique_ptr<ECombine> K(new ECombine());
      memset(&K->p, 0, sizeof(K->p));
      int n = 0;
      for (int idx = 0; idx < 3 && node_in[i][idx] >= 0; ++idx, ++n) {
        const int o = node_in[i][idx];
        Planes src = maybe_1x1(c, feats[o], pre + "/resample_" + std::to_string(idx) + "_" + std::to_string(o) + "_" +
                                                 std::to_string(nfeats));
        if (set_input(K->p.in[idx], src, th, tw)) return -1;
        K->wnames[idx] = pre + "/WSM" + (idx == 0 ? std::string() : "_" + std::to_string(idx));
      }
      Planes comb = c->planes(th, tw, c->Fp, c->F);
      K->p.n_in = n; K->p.B = c->B; K->p.Ho = th; K->p.Wo = tw; K->p.C = c->Fp;
      K->p.weighted = g.fpn_weight_method == 1; K->p.denom = 1.f; K->p.swish = 1;
      K->p.out_hi = comb.hi; K->p.out_lo = comb.lo;
      add_combine(c, std::move(K));
      const std::string op = pre + "/op_after_combine" + std::to_string(nfeats);
      Planes t = c->planes(th, tw, c->Fp, c->F);
      add_dw(c, op + "/conv/depthwise_kernel", comb, t);
      Planes node = c->planes(th, tw, c->Fp, c->F);
      add_pw(c, op + "/conv/pointwise_kernel", op + "/conv/bias", op + "/bn", t, node, c->F, 0);
      feats.push_back(node);
    }
    // the cell's outputs: the last node of every level (arch.py:495-503)
    std::vector<Planes> next(5);
    for (int l = 3; l <= 7; ++l)
      for (int i = 7; i >= 0; --i)
        if (node_level[i] == l) { next[l - 3] = feats[feats.size() - 8 + i]; break; }
    feats = next;
  }
  for (int l = 0; l < 5; ++l) {
    c->fpn_out[l] = feats[l];
    c->named.planes("fpn" + std::to_string(l + 3), feats[l]);
  }
  // class / box nets (arch.py:227-340), writing the post-processing inputs
  EffdetPostParams& p = c->post;
  memset(&p, 0, sizeof(p));
  const int ncls = c->na * g.num_classes, nbox = c->na * 4;
  for (int l = 0; l < 5; ++l) {
    const int level = l + 3, h = c->fh[level], w = c->fw[level];
    for (int kind = 0; kind < 2; ++kind) {
      const std::string kn = kind == 0 ? "class" : "box";
      Planes x = c->fpn_out[l];
      Planes ping = c->planes(h, w, c->Fp, c->F), pong = c->planes(h, w, c->Fp, c->F), t = c->planes(h, w, c->Fp, c->F);
      for (int i = 0; i < g.box_class_repeats; ++i) {
        const std::string nm = kn + "_net/" + kn + "-" + std::to_string(i);
        add_dw(c, nm + "/depthwise_kernel", x, t);
        Planes y = (i & 1) ? pong : ping;
        add_pw(c, nm + "/pointwise_kernel", nm + "/bias", nm + "-bn-" + std::to_string(level), t, y, c->F, 2);
        x = y;
      }
      const std::string nm = kn + "_net/" + kn + "-predict";
      add_dw(c, nm + "/depthwise_kernel", x, t);
      const int creal = kind == 0 ? ncls : nbox, ld = pad16(creal);
      float* o = c->arena.alloc<float>(static_cast<size_t>(c->B) * h * w * ld);
      add_pw(c, nm + "/pointwise_kernel", nm + "/bias", "", t, Planes(), creal, 0, nullptr, o, ld);
      (kind == 0 ? p.logits[l] : p.boxes[l]) = o;
      (kind == 0 ? p.ld[l] : p.ldb[l]) = ld;
      (kind == 0 ? p.logit_bstride[l] : p.box_bstride[l]) = static_cast<unsigned long long>(h) * w * ld;
      c->named.raw((kind == 0 ? "cls" : "box") + std::to_string(level), o, Stage::kF32, c->B, h, w, ld);
    }
  }
  // post-processing state
  unsigned long long off = 0;
  for (int l = 0; l < 5; ++l) {
    const int level = l + 3;
    p.w[l] = c->fw[level];
    p.level_off[l] = off;
    off += static_cast<unsigned long long>(c->fh[level]) * c->fw[level] * ncls;
    // anchors.py:216-257: stride = image / feature size; octave scale 2^(o / num_scales); aspect (x, y) multipliers
    p.stride_y[l] = static_cast<double>(g.image_h) / c->fh[level];
    p.stride_x[l] = static_cast<double>(g.image_w) / c->fw[level];
    int a = 0;
    for (int o = 0; o < g.num_scales; ++o)
      for (int r = 0; r < g.num_aspects; ++r, ++a) {
        const double oct = pow(2.0, o / static_cast<double>(g.num_scales));
        const double sx = config_double(g.anchor_scale) * p.stride_x[l] * oct;
        const double sy = config_double(g.anchor_scale) * p.stride_y[l] * oct;
        p.half_x[l][a] = sx * config_double(g.aspect_ratios[r][0]) / 2.0;
        p.half_y[l][a] = sy * config_double(g.aspect_ratios[r][1]) / 2.0;
      }
  }
  p.level_off[5] = off; p.total = off;
  p.n_levels = 5; p.anchors = c->na; p.num_classes = g.num_classes; p.min_level = 3;
  p.k = g.max_detection_topk; p.max_out = g.result_per_im;
  B2_CHECK(p.k >= 1 && p.k <= 8192, "effdet: max_detection_topk must be in [1, 8192]");
  p.score_thresh = g.result_score_thres; p.nms_thr = g.nms_iou_threshold;
  // one slice per image of the scratch and the outputs
  const size_t B = static_cast<size_t>(c->B), kb = B * p.k, mb = B * p.max_out;
  p.B = c->B;
  p.hist = c->arena.alloc<unsigned int>(B * 256);
  p.state = c->arena.alloc<uint32_t>(B * 8);
  p.cand = c->arena.alloc<unsigned long long>(kb);
  p.ties = c->arena.alloc<unsigned long long>(kb);
  p.tie_cnt = c->arena.alloc<unsigned int>(B * effdet_topk_blocks());
  p.tie_off = c->arena.alloc<unsigned int>(B * effdet_topk_blocks());
  p.cand_box = c->arena.alloc<float4>(kb);
  p.cand_score = c->arena.alloc<float>(kb);
  p.cand_cls = c->arena.alloc<int>(kb);
  p.cand_lvl = c->arena.alloc<int>(kb);
  p.mask = c->arena.alloc<unsigned long long>(kb * ((p.k + 63) / 64));
  c->out_boxes = c->arena.alloc<float4>(mb);
  c->out_scores = c->arena.alloc<float>(mb);
  c->out_classes = c->arena.alloc<int>(mb);
  c->out_levels = c->arena.alloc<int>(mb);
  c->out_count = c->arena.alloc<int>(B);
  c->out_feat = c->arena.alloc<float>(mb * c->F);
  c->scale_dev = c->arena.alloc<float>(B);
  p.out_boxes = c->out_boxes; p.out_scores = c->out_scores; p.out_classes = c->out_classes;
  p.out_levels = c->out_levels; p.out_count = c->out_count;
  LevelRoiFeatParams& r = c->roi;
  memset(&r, 0, sizeof(r));
  for (int l = 0; l < 5; ++l) {
    r.feat_hi[l] = c->fpn_out[l].hi; r.feat_lo[l] = c->fpn_out[l].lo;
    r.H[l] = c->fpn_out[l].H; r.W[l] = c->fpn_out[l].W;
    r.inv_stride[l] = 1.0f / static_cast<float>(1 << (l + 3));
  }
  r.B = c->B; r.C = c->Fp; r.Creal = c->F; r.min_level = 3; r.max_out = p.max_out;
  r.boxes = c->out_boxes; r.levels = c->out_levels; r.count = c->out_count; r.out = c->out_feat;
  // the candidates in top-k order (boxes ymin xmin ymax xmax in network pixels, count = state[5]), the outputs, and the
  // device copy of image_scale the NMS step multiplies the boxes by; shape[0] = the batch
  const int k = p.k, m = p.max_out, nb = c->B;
  c->named.raw("topk_boxes", p.cand_box, Stage::kF32, nb, 1, k, 4);
  c->named.raw("topk_scores", p.cand_score, Stage::kF32, nb, 1, k, 1);
  c->named.raw("topk_classes", p.cand_cls, Stage::kI32, nb, 1, k, 1);
  c->named.raw("topk_levels", p.cand_lvl, Stage::kI32, nb, 1, k, 1);
  if (nb == 1) c->named.raw("topk_count", p.state + 5, Stage::kI32, 1, 1, 1, 1);
  else c->named.raw("topk_count", p.state, Stage::kI32, nb, 1, 1, 8);   // [B][8]: the count is column 5
  c->named.raw("final_boxes", c->out_boxes, Stage::kF32, nb, 1, m, 4);
  c->named.raw("final_scores", c->out_scores, Stage::kF32, nb, 1, m, 1);
  c->named.raw("final_classes", c->out_classes, Stage::kI32, nb, 1, m, 1);
  c->named.raw("final_levels", c->out_levels, Stage::kI32, nb, 1, m, 1);
  c->named.raw("final_count", c->out_count, Stage::kI32, nb, 1, 1, 1);
  c->named.raw("box_feat", c->out_feat, Stage::kF32, nb, 1, m, c->F);
  c->named.raw("image_scale", c->scale_dev, Stage::kF32, nb, 1, 1, 1);
  // 15 kernels (seed, 4 x (hist, pick), collect, tie scan, tie write, prepare, mask, scan), counted as the 14 that
  // b2_effdet_num_launches has always reported for them; every one covers all images
  add_step(c->steps, kPost, 6, "post", [c](cudaStream_t st) { return effdet_post_launch(c->post, c->scale_dev, st); },
           static_cast<double>(p.total) * 4.0 * 6.0 * c->B, 0.0, 14);
  add_step(c->steps, kBoxFeat, 7, "box_feat", [c](cudaStream_t st) { return level_roi_feat_launch(c->roi, st); }, 0.0);
  B2_CHECK(c->arena.failed() == 0,
           "b2_effdet_create: out of device memory: a batch-" + std::to_string(c->B) + " context needs " +
               std::to_string(c->arena.requested()) + " bytes of device memory, and " + std::to_string(c->arena.failed()) +
               " of them could not be allocated");
  return plan_convs(c->convs, c->split, c->num_sms);
}


// Runs the pass on the images as they stand (image_scale[B] of every image) and copies images [0, n) of the outputs.
int launch_and_fetch(b2_effdet* c, bool full, const float* image_scale, int n, float* boxes, float* scores, int* classes,
                     int* levels, float* box_feat, int* count) {
  B2_CUDA(cudaMemcpyAsync(c->scale_dev, image_scale, sizeof(float) * c->B, cudaMemcpyHostToDevice, c->stream));
  cudaGraphExec_t& graph = full ? c->graph_full : c->graph;
  const unsigned mask = full ? ~0u : ~(1u << kBackbone);
  if (!graph && capture_graph(c->stream, [c, mask] { return run_steps(c->steps, mask, c->stream); }, &graph)) return -1;
  B2_CUDA(cudaGraphLaunch(graph, c->stream));
  const size_t m = static_cast<size_t>(n) * c->post.max_out;
  B2_CUDA(cudaMemcpyAsync(boxes, c->out_boxes, sizeof(float) * 4 * m, cudaMemcpyDeviceToHost, c->stream));
  B2_CUDA(cudaMemcpyAsync(scores, c->out_scores, sizeof(float) * m, cudaMemcpyDeviceToHost, c->stream));
  B2_CUDA(cudaMemcpyAsync(classes, c->out_classes, sizeof(int) * m, cudaMemcpyDeviceToHost, c->stream));
  if (levels) B2_CUDA(cudaMemcpyAsync(levels, c->out_levels, sizeof(int) * m, cudaMemcpyDeviceToHost, c->stream));
  if (box_feat) B2_CUDA(cudaMemcpyAsync(box_feat, c->out_feat, sizeof(float) * m * c->F, cudaMemcpyDeviceToHost, c->stream));
  B2_CUDA(cudaMemcpyAsync(count, c->out_count, sizeof(int) * n, cudaMemcpyDeviceToHost, c->stream));
  B2_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

// Uploads frames [0, n) back to back into the grow-only frame buffer, pre-processes them into images [0, n) and the last
// frame again into images [n, B) (a short batch is padded as the reference's batch driver pads it, so one graph serves
// every n), then runs the whole pass.  image_scale_out[i] = image_scale_to_original of frame i.
int detect_frames(b2_effdet* c, const char* who, const uint8_t* const* frames, const int* h, const int* w, int n,
                  float* boxes, float* scores, int* classes, int* levels, float* box_feat, int* count,
                  float* image_scale_out) {
  B2_CUDA(cudaSetDevice(c->device));
  B2_CHECK(c->loaded, std::string(who) + ": weights not loaded");
  B2_CHECK(c->cfg.backbone >= 0,
           std::string(who) + ": the context was created without a backbone (use b2_effdet_run_features)");
  std::vector<unsigned long long> off(n);
  size_t bytes = 0;
  for (int i = 0; i < n; ++i) {
    B2_CHECK(frames[i], std::string(who) + ": null frame");
    B2_CHECK(h[i] >= 1 && w[i] >= 1, std::string(who) + ": empty frame");
    off[i] = bytes;
    bytes += static_cast<size_t>(h[i]) * w[i] * 3;
  }
  if (bytes > c->frame_cap) {
    if (c->frame) B2_CUDA(cudaFree(c->frame));
    c->frame = nullptr; c->frame_cap = 0;
    B2_CUDA(cudaMalloc(&c->frame, bytes));
    c->frame_cap = bytes;
  }
  std::vector<EffnetFrame> table(c->B);
  std::vector<float> scales(c->B);
  for (int b = 0; b < c->B; ++b) {
    const int i = b < n ? b : n - 1;
    // set_scale_factors_to_output_size (dataloader.py:101-113), float32 like the TF graph
    const float sy = static_cast<float>(c->cfg.image_h) / static_cast<float>(h[i]);
    const float sx = static_cast<float>(c->cfg.image_w) / static_cast<float>(w[i]);
    const float scale = sx < sy ? sx : sy;
    int sh = static_cast<int>(static_cast<float>(h[i]) * scale), sw = static_cast<int>(static_cast<float>(w[i]) * scale);
    if (sh > c->cfg.image_h) sh = c->cfg.image_h;
    if (sw > c->cfg.image_w) sw = c->cfg.image_w;
    B2_CHECK(sh >= 1 && sw >= 1, std::string(who) + ": frame " + std::to_string(i) + " resizes to an empty image");
    table[b] = effnet_frame(off[i], h[i], w[i], sh, sw);
    scales[b] = 1.0f / scale;
  }
  for (int i = 0; i < n; ++i) {
    B2_CUDA(cudaMemcpyAsync(c->frame + off[i], frames[i], static_cast<size_t>(h[i]) * w[i] * 3, cudaMemcpyHostToDevice,
                            c->stream));
    if (image_scale_out) image_scale_out[i] = scales[i];
  }
  B2_CUDA(cudaMemcpyAsync(c->frame_table, table.data(), sizeof(EffnetFrame) * c->B, cudaMemcpyHostToDevice, c->stream));
  if (effnet_preprocess_launch(c->frame, c->frame_table, c->B, c->image, c->cfg.image_h, c->cfg.image_w, c->stream))
    return -1;
  return launch_and_fetch(c, true, scales.data(), n, boxes, scores, classes, levels, box_feat, count);
}

}  // namespace

extern "C" {

int b2_effdet_create(b2_effdet** out, const b2_effdet_config* cfg, int device) {
  B2_CHECK(out && cfg, "b2_effdet_create: null argument");
  *out = nullptr;
  std::unique_ptr<b2_effdet> c(new b2_effdet());
  B2_CHECK(cfg->batch >= 0 && cfg->batch <= 1024, "b2_effdet_create: batch must be in [0, 1024] (0 means 1)");
  c->cfg = *cfg; c->device = device; c->split = cfg->precision == 1;
  c->B = cfg->batch > 1 ? cfg->batch : 1;
  if (open_device(device, "b2_effdet_create", &c->num_sms, &c->stream)) return -1;
  if (build(c.get())) { b2_effdet_destroy(c.release()); return -1; }
  B2_CUDA(cudaDeviceSynchronize());
  *out = c.release();
  return 0;
}

void b2_effdet_destroy(b2_effdet* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  if (c->graph) cudaGraphExecDestroy(c->graph);
  if (c->graph_full) cudaGraphExecDestroy(c->graph_full);
  if (c->frame) cudaFree(c->frame);
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;   // plans, then the arena's device memory
}

// TF checkpoint variables of the feature network and heads (names as in efficientdet_arch.py, kernels HWIO)
int b2_effdet_load_weights(b2_effdet* c, const char* const* names, const float* const* data, const int64_t* numel, int n) {
  B2_CHECK(c && names && data && numel, "b2_effdet_load_weights: null argument");
  B2_CUDA(cudaSetDevice(c->device));
  const WeightSet ws(names, data, numel, n);
  for (auto& L : c->convs) {
    const int K = L->w.K, Cp = L->w.Cout_pad, co = L->d.Cout, ci = L->cin_real;
    const float* w = ws.get(L->name, static_cast<int64_t>(ci) * co);
    const float* b = L->bias.empty() ? nullptr : ws.get(L->bias, co);   // backbone convs have no bias
    if (!w || (!b && !L->bias.empty())) return -1;
    std::vector<double> scale, shift;
    if (fold_bn(ws, L->bn, kKerasBn, 1e-3, co, scale, shift)) return -1;   // utils.py:252-303 eps
    std::vector<float> packed(static_cast<size_t>(Cp) * K, 0.f);
    for (int o = 0; o < co; ++o)
      for (int i = 0; i < ci; ++i) packed[static_cast<size_t>(o) * K + i] = static_cast<float>(w[static_cast<size_t>(i) * co + o] * scale[o]);
    if (upload_conv(*L, packed, fold_bias(scale, shift, b, co, Cp), c->stream)) return -1;
  }
  for (auto& kv : c->dw_shared) {
    const int C = c->Fp, cr = c->F;
    const float* w = ws.get(kv.first, static_cast<int64_t>(9) * cr);   // [3,3,C,1]
    if (!w) return -1;
    std::vector<float> pw(9 * static_cast<size_t>(C), 0.f);
    for (int t = 0; t < 9; ++t)
      for (int ch = 0; ch < cr; ++ch) pw[static_cast<size_t>(t) * C + ch] = w[t * cr + ch];
    B2_CUDA(cudaMemcpyAsync(kv.second, pw.data(), pw.size() * 4, cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
  }
  for (auto& D : c->dwbns) {
    const int C = D->p.C, cr = D->creal, kk = D->p.K * D->p.K;
    const float* w = ws.get(D->wname, static_cast<int64_t>(kk) * cr);   // [K,K,C,1]
    std::vector<double> scale, shift;
    if (!w || fold_bn(ws, D->bnname, kKerasBn, 1e-3, cr, scale, shift)) return -1;
    std::vector<float> pw(static_cast<size_t>(kk) * C, 0.f), pb(C, 0.f);
    for (int ch = 0; ch < cr; ++ch) {
      for (int t = 0; t < kk; ++t) pw[static_cast<size_t>(t) * C + ch] = static_cast<float>(w[t * cr + ch] * scale[ch]);
      pb[ch] = static_cast<float>(shift[ch]);
    }
    B2_CUDA(cudaMemcpyAsync(D->w, pw.data(), pw.size() * 4, cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaMemcpyAsync(D->bias, pb.data(), pb.size() * 4, cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
  }
  for (auto& S : c->ses) {
    const int m = S->creal, r = S->nr;
    const float* w1 = ws.get(S->pre + "/conv2d/kernel", static_cast<int64_t>(m) * r);
    const float* b1 = ws.get(S->pre + "/conv2d/bias", r);
    const float* w2 = ws.get(S->pre + "/conv2d_1/kernel", static_cast<int64_t>(r) * m);
    const float* b2 = ws.get(S->pre + "/conv2d_1/bias", m);
    if (!w1 || !b1 || !w2 || !b2) return -1;
    B2_CUDA(cudaMemcpyAsync(S->w1, w1, sizeof(float) * m * r, cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaMemcpyAsync(S->b1, b1, sizeof(float) * r, cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaMemcpyAsync(S->w2, w2, sizeof(float) * r * m, cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaMemcpyAsync(S->b2, b2, sizeof(float) * m, cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
  }
  if (c->cfg.fpn_weight_method == 1) {
    for (auto& K : c->combines) {
      if (!K->p.weighted) continue;
      float raw[3];
      for (int i = 0; i < K->p.n_in; ++i) {
        const float* w = ws.get(K->wnames[i], 1);
        if (!w) return -1;
        raw[i] = w[0];
      }
      bifpn_set_weights(K->p, raw);
    }
  }
  c->loaded = true;
  if (c->graph) { cudaGraphExecDestroy(c->graph); c->graph = nullptr; }
  if (c->graph_full) { cudaGraphExecDestroy(c->graph_full); c->graph_full = nullptr; }
  return 0;
}

// Backbone features C3, C4, C5 as host NHWC fp32 ([h,w,c] with the real channel counts) -> detections.
// boxes [max][4] x1 y1 x2 y2 in original-frame pixels (network coords * image_scale), classes 1-based, levels 3..7,
// box_feat [max][fpn_num_filters].  Returns the number of detections in *count (rows beyond it are zero).
int b2_effdet_run_features(b2_effdet* c, const float* c3, const float* c4, const float* c5, float image_scale,
                           float* boxes, float* scores, int* classes, int* levels, float* box_feat, int* count) {
  B2_CHECK(c && c3 && c4 && c5 && boxes && scores && classes && count, "b2_effdet_run_features: null argument");
  B2_CUDA(cudaSetDevice(c->device));
  B2_CHECK(c->loaded, "b2_effdet_run_features: weights not loaded");
  B2_CHECK(c->B == 1, "b2_effdet_run_features: the context was created for a batch of " + std::to_string(c->B) +
                          " images and this call takes one image's features; use a batch-1 context");
  const float* src[3] = {c3, c4, c5};
  for (int i = 0; i < 3; ++i) {
    const Planes& p = c->backbone[i];
    std::vector<float> padded(p.elems(), 0.f);
    const size_t px = static_cast<size_t>(p.H) * p.W;
    for (size_t q = 0; q < px; ++q) memcpy(&padded[q * p.C], src[i] + q * p.creal, sizeof(float) * p.creal);
    if (upload_planes(padded.data(), p.hi, p.lo, padded.size(), c->stream)) return -1;
  }
  return launch_and_fetch(c, false, &image_scale, 1, boxes, scores, classes, levels, box_feat, count);
}

// Full per-frame path of the reference wrapper (EfficientDet.build_preprocess + build_model): host BGR uint8 frame
// [h,w,3] -> pre-process (RGB, /255, mean/std, bilinear resize to fit, zero-pad) -> backbone -> BiFPN -> heads ->
// detections scaled back to the frame.  *image_scale_out = image_scale_to_original.
int b2_effdet_detect(b2_effdet* c, const uint8_t* frame_bgr, int h, int w, float* boxes, float* scores, int* classes,
                     int* levels, float* box_feat, int* count, float* image_scale_out) {
  B2_CHECK(c && frame_bgr && boxes && scores && classes && count, "b2_effdet_detect: null argument");
  B2_CHECK(h >= 1 && w >= 1, "b2_effdet_detect: empty frame");
  B2_CHECK(c->B == 1, "b2_effdet_detect: the context was created for a batch of " + std::to_string(c->B) +
                          " images; use b2_effdet_detect_batch");
  return detect_frames(c, "b2_effdet_detect", &frame_bgr, &h, &w, 1, boxes, scores, classes, levels, box_feat, count,
                       image_scale_out);
}

// The same for 1 <= n <= batch frames of any sizes in one pass: image i's outputs at row block i of boxes [batch][max][4],
// scores / classes / levels [batch][max], box_feat [batch][max][F], counts [batch], image_scales [batch]; blocks i >= n
// are not written.
int b2_effdet_detect_batch(b2_effdet* c, const uint8_t* const* frames, const int* h, const int* w, int n, float* boxes,
                           float* scores, int* classes, int* levels, float* box_feat, int* counts, float* image_scales) {
  B2_CHECK(c && frames && h && w && boxes && scores && classes && counts, "b2_effdet_detect_batch: null argument");
  B2_CHECK(n >= 1 && n <= c->B, "b2_effdet_detect_batch: n = " + std::to_string(n) + " frames, the context takes 1 to " +
                                    std::to_string(c->B));
  return detect_frames(c, "b2_effdet_detect_batch", frames, h, w, n, boxes, scores, classes, levels, box_feat, counts,
                       image_scales);
}

// Stage-addressable tensors of the last pass as fp32 NHWC: "fpn3".."fpn7" (BiFPN outputs, channel-padded),
// "cls3".."cls7" / "box3".."box7" (head outputs, row stride = shape[3] >= real columns).
int b2_effdet_get_stage(b2_effdet* c, const char* name, float* dst, int64_t capacity, int64_t shape[4]) {
  B2_CHECK(c && name && dst && shape, "b2_effdet_get_stage: null argument");
  B2_CUDA(cudaSetDevice(c->device));
  return stage_get(c->named, name, c->stream, dst, capacity, shape, "b2_effdet_get_stage");
}

// Overwrites stage `name` with host data of its full stored shape (4 bytes per element), e.g. "cls3".."cls7" /
// "box3".."box7" with their padding columns and "fpn3".."fpn7" with their padded channels, so that the phases after it can
// run on chosen inputs.
int b2_effdet_set_stage(b2_effdet* c, const char* name, const void* src, int64_t bytes) {
  B2_CHECK(c && name && src, "b2_effdet_set_stage: null argument");
  B2_CUDA(cudaSetDevice(c->device));
  const Stage* s = c->named.find(name);
  if (!s) return -1;
  B2_CHECK(bytes == s->numel() * 4, "b2_effdet_set_stage: size mismatch");
  return stage_write(*s, c->stream, src);
}

// Runs the steps of the phases in `mask` (B2_EFFDET_PHASE_*) eagerly on the stages as they stand, and waits for them.
int b2_effdet_run_phases(b2_effdet* c, int mask) {
  B2_CHECK(c, "b2_effdet_run_phases: null argument");
  B2_CUDA(cudaSetDevice(c->device));
  B2_CHECK(c->loaded, "b2_effdet_run_phases: weights not loaded");
  B2_CHECK(!(mask & (1 << kBackbone)) || c->cfg.backbone >= 0, "b2_effdet_run_phases: the context has no backbone");
  if (run_steps(c->steps, static_cast<unsigned>(mask), c->stream)) return -1;
  B2_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

// Per-step CUDA-event timing of the whole pass (backbone when present, feature network, heads, post-processing, box
// feature), eager launches on the context stream.  ms_out[i] = mean over `reps` of step i; *n_out = number of steps.
int b2_effdet_profile_steps(b2_effdet* c, int reps, float* ms_out, int cap, int* n_out) {
  B2_CHECK(c && ms_out && n_out && reps >= 1, "b2_effdet_profile_steps: bad argument");
  B2_CUDA(cudaSetDevice(c->device));
  B2_CHECK(c->loaded, "b2_effdet_profile_steps: weights not loaded");
  return profile_steps(c->steps, c->stream, reps, ms_out, cap, n_out);
}

// Step `idx` of b2_effdet_profile_steps: kind (0 pointwise conv on the tensor cores, 1 head/BiFPN depthwise, 2 BiFPN
// combine / max-pool, 3 backbone depthwise, 4 squeeze-excite, 5 stem im2col, 6 post-processing, 7 box feature), a
// name, algorithmic FLOPs and HBM bytes (operands once, at the stored precision).
int b2_effdet_step_info(b2_effdet* c, int idx, char* name, int name_cap, double* flops, double* bytes, int* kind) {
  B2_CHECK(c, "b2_effdet_step_info: null argument");
  return step_info(c->steps, idx, name, name_cap, flops, bytes, kind);
}

// Replays the whole-frame graph that b2_effdet_detect / b2_effdet_detect_batch captured `reps` times on the images as
// they stand, with no host copies; *ms_out = mean milliseconds per replay (CUDA events).
int b2_effdet_replay(b2_effdet* c, int reps, float* ms_out) {
  B2_CHECK(c && ms_out && reps >= 1, "b2_effdet_replay: bad argument");
  B2_CUDA(cudaSetDevice(c->device));
  B2_CHECK(c->graph_full, "b2_effdet_replay: no captured graph yet (run b2_effdet_detect or b2_effdet_detect_batch first)");
  cudaEvent_t ev[2] = {nullptr, nullptr};
  B2_CUDA(cudaEventCreate(&ev[0]));
  if (cudaEventCreate(&ev[1]) != cudaSuccess) {
    cudaEventDestroy(ev[0]);
    B2_CHECK(false, "b2_effdet_replay: cudaEventCreate failed");
  }
  cudaError_t e = cudaEventRecord(ev[0], c->stream);
  for (int r = 0; r < reps && e == cudaSuccess; ++r) e = cudaGraphLaunch(c->graph_full, c->stream);
  if (e == cudaSuccess) e = cudaEventRecord(ev[1], c->stream);
  if (e == cudaSuccess) e = cudaEventSynchronize(ev[1]);
  float ms = 0.f;
  if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, ev[0], ev[1]);
  cudaEventDestroy(ev[0]);
  cudaEventDestroy(ev[1]);
  B2_CUDA(e);
  *ms_out = ms / reps;
  return 0;
}

// Kernels of one b2_effdet_detect call (pre-processing + the whole pass); b2_effdet_run_features runs the steps after the
// backbone.
int b2_effdet_num_launches(b2_effdet* c) {
  if (!c) return -1;
  return total_launches(c->steps) + (c->cfg.backbone >= 0 ? 1 : 0);   // + pre-processing
}

}  // extern "C"
