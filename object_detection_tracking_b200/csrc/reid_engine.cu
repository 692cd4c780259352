// OSNet-x1.0 ReID embedding engine (torchreid FeatureExtractor replacement) and the distance-matrix
// GEMM, behind the C ABI.  One b2_reid = one device = one fixed crop batch; the pass is a fixed launch
// sequence replayed as a CUDA graph.
//
// Reference graph: torchreid/models/osnet.py OSNet.forward (:413-438) with osnet_x1_0 (:522-534):
//   conv1 7x7/2 + BN + ReLU -> maxpool 3/2 -> [OSBlock x2 + Conv1x1 + AvgPool2] x2 -> OSBlock x2 -> conv5 1x1
//   -> global avg-pool -> fc(512) + BatchNorm1d + ReLU  (eval mode returns this 512-d vector)
// Input contract (torchreid/feature_extractor.py:190-196,209-252): RGB uint8 crops already resized to
// 256x128 (b2_reid_embed: the caller ran the PIL resize), or uint8 BGR frames plus a table of track boxes
// (b2_reid_embed_boxes: reid_ingest.cu cuts and resizes them as Pillow does into the same crop buffer); ToTensor +
// Normalize happen in the stem pack kernel.
//
// Second model (b2_reid_create_model(..., model = 1)): torchreid's resnet101 (torchreid/models/resnet.py:441-455 ->
// ResNet(Bottleneck, [3, 4, 23, 3], last_stride=2, fc_dims=None), forward :342-366), the vehicle extractor of
// single_video_reid.py:410-415 with image_size (128, 256):  conv1 7x7/2 + BN + ReLU -> maxpool 3/2 pad 1 ->
// layer1..4 of Bottleneck blocks (1x1 -> 3x3 carrying the stride -> 1x1, BN folded, ReLU / residual in the epilogue,
// 1x1 strided downsample on the first block of a layer) -> global avg-pool = the 2048-d feature (eval mode).
// Every conv runs on conv_tc_kernel (wgmma); max-pool / global-average kernels are shared with OSNet.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <memory>
#include <string>
#include <vector>

#include "../../include/b200det.h"
#include "engine_core.h"
#include "kernels.h"

using namespace b2;

namespace {

struct RDw {
  std::string wname, bnname;
  Planes in, out;
  float* w = nullptr;      // [9][C]
  float* bias = nullptr;   // [C]
  int creal = 0;
};

struct RGate {
  std::string prefix;      // "...gate"
  Planes s[4], out;
  float *pooled = nullptr, *gates = nullptr, *w1 = nullptr, *b1 = nullptr, *w2 = nullptr, *b2 = nullptr;
  int creal = 0, cr = 0;
};

// ConvLayer::layout: how the torch weight is packed
enum { kOI = 0, kStem = 1, kOIHW = 2 };   // [O][I] (1x1 OIHW or Linear), packed 7x7 stem, RxS conv OIHW

}  // namespace

struct b2_reid {
  Arena arena;                       // first member: freed after everything that refers to it
  int device = 0, num_sms = 132, B = 0;
  int model = 0;                     // 0 osnet_x1_0, 1 resnet101
  int in_h = 256, in_w = 128;        // crop size (h, w) the extractor resizes to
  int feat_dim = 512;
  bool split = true;
  cudaStream_t stream = nullptr;
  std::vector<std::unique_ptr<ConvLayer>> convs;
  std::vector<std::unique_ptr<RDw>> dws;
  std::vector<std::unique_ptr<RGate>> gates;
  std::vector<Step> steps;
  StageMap named;                    // stage-addressable activations (parity tests)
  uint8_t* crops = nullptr;          // [B][in_h][in_w][3] RGB, the stem pack's input
  uint8_t* frames = nullptr;         // b2_reid_embed_boxes: uploaded frames, grow-only (cudaMalloc, freed on destroy)
  size_t frames_cap = 0;
  int32_t* boxes = nullptr;          // [B][5] box table of the last b2_reid_embed_boxes call
  Planes stem_u, gap_planes;
  float* gap_f32 = nullptr;
  float* feats = nullptr;      // [Bpad][512]
  cudaGraphExec_t graph = nullptr;
  bool loaded = false;

  Planes planes(int b, int h, int w, int c) { return arena.planes(b, h, w, c, split); }
};

namespace {

int pad64(int c) { return (c + 63) / 64 * 64; }

// k x k conv (torch Conv2d, symmetric padding; dense layers as 1x1) in -> out planes, or -> fp32 rows of stride ldc32,
// with optional BN / bias / ReLU / residual
ConvLayer* add_conv(b2_reid* c, const std::string& wname, const std::string& bn, const std::string& bias, const Planes& in,
                    int cin_real, const Planes& out, int cout_real, bool relu, const Planes* res, int k = 1, int stride = 1,
                    int pad = 0, float* out_f32 = nullptr, int ldc32 = 0) {
  ConvDesc d;
  d.R = d.S = k; d.stride = stride;
  d.pad_t = d.pad_l = pad;
  // stride 2 on even extents: the last window ends one row / column before torch's bottom / right padding, so
  // (pad, pad - 1) is the same convolution -- and exactly the geometry the detector's strided layers use
  // (nn.py:487-492 3x3 with pads (1,0); :555-560 1x1 with the last row / column dropped).
  d.pad_b = d.pad_r = stride == 2 ? pad - 1 : pad;
  d.Cout = cout_real; d.relu = relu ? 1 : 0;
  std::unique_ptr<ConvLayer> L = make_conv(c->arena, c->split, wname, d, in, out, res, out_f32, ldc32);
  L->bn = bn; L->bias = bias; L->cin_real = cin_real;
  L->layout = (k != 1 || stride != 1) ? kOIHW : kOI;
  ConvLayer* raw = L.get();
  add_conv_step(c->steps, 0, raw);
  c->convs.push_back(std::move(L));
  return raw;
}

// conv1 7x7/2 pad 3 through the packed-operand trick of stem.cu: a 4x1 VALID conv over the packed operand
Planes add_stem(b2_reid* c, const std::string& wname, const std::string& bn) {
  const int B = c->B, h1 = (c->in_h + 6 - 7) / 2 + 1, w1 = (c->in_w + 6 - 7) / 2 + 1;
  c->stem_u = c->planes(B, h1 + 3, w1, 64);
  const Planes u = c->stem_u;
  add_step(c->steps, 0, 0, "", [c, u](cudaStream_t st) {
    return stem_pack_launch(c->crops, c->B, c->in_h, c->in_w, u.hi, u.lo, u.H, u.W, st);
  });
  Planes c1 = c->planes(B, h1, w1, 64);
  ConvDesc d;
  d.R = 4; d.S = 1; d.Cout = 64; d.relu = 1;
  std::unique_ptr<ConvLayer> L = make_conv(c->arena, c->split, wname, d, c->stem_u, c1);
  L->bn = bn; L->cin_real = 64; L->layout = kStem;
  add_conv_step(c->steps, 0, L.get());
  c->convs.push_back(std::move(L));
  c->named.planes("stem_u", c->stem_u);
  c->named.planes("conv1", c1);
  return c1;
}

// maxpool 3/2 pad 1: nn.MaxPool2d(3, 2, 1) gives (H - 1) / 2 + 1 rows, the last window cut by the border when H is odd
Planes add_maxpool(b2_reid* c, const Planes& a) {
  const Planes b = c->planes(a.B, (a.H - 1) / 2 + 1, (a.W - 1) / 2 + 1, a.C);
  add_step(c->steps, 0, 0, "", [a, b](cudaStream_t st) {
    return maxpool_launch(a.hi, a.lo, a.B, a.H, a.W, a.C, b.hi, b.lo, b.H, b.W, st);
  });
  c->named.planes("maxpool", b);
  return b;
}

Planes add_light(b2_reid* c, const std::string& pre, const Planes& in, int creal) {
  // LightConv3x3 (osnet.py:128-156): 1x1 linear (no BN) -> depthwise 3x3 -> BN -> ReLU
  Planes t = c->planes(in.B, in.H, in.W, in.C);
  add_conv(c, pre + ".conv1.weight", "", "", in, creal, t, creal, false, nullptr);
  std::unique_ptr<RDw> D(new RDw());
  D->wname = pre + ".conv2.weight"; D->bnname = pre + ".bn";
  D->in = t; D->out = c->planes(in.B, in.H, in.W, in.C);
  D->w = c->arena.alloc<float>(9 * in.C); D->bias = c->arena.alloc<float>(in.C);
  D->creal = creal;
  const RDw* dw = D.get();
  add_step(c->steps, 0, 0, "", [dw](cudaStream_t st) {
    return dwconv3x3_launch(dw->in.hi, dw->in.lo, dw->in.B, dw->in.H, dw->in.W, dw->in.C, dw->w, dw->bias, dw->out.hi,
                            dw->out.lo, st);
  });
  c->dws.push_back(std::move(D));
  return dw->out;
}

Planes add_osblock(b2_reid* c, const std::string& pre, const Planes& x, int cin, int cout) {
  // OSBlock (osnet.py:223-276)
  const int mid = cout / 4, midp = pad64(mid);
  Planes x1 = c->planes(x.B, x.H, x.W, midp);
  add_conv(c, pre + ".conv1.conv.weight", pre + ".conv1.bn", "", x, cin, x1, mid, true, nullptr);
  Planes s[4];
  const char* names[4] = {".conv2a", ".conv2b", ".conv2c", ".conv2d"};
  for (int k = 0; k < 4; ++k) {
    Planes t = x1;
    if (k == 0) t = add_light(c, pre + names[k], t, mid);
    else
      for (int j = 0; j <= k; ++j) t = add_light(c, pre + names[k] + "." + std::to_string(j), t, mid);
    s[k] = t;
  }
  std::unique_ptr<RGate> G(new RGate());
  G->prefix = pre + ".gate";
  for (int k = 0; k < 4; ++k) G->s[k] = s[k];
  G->out = c->planes(x.B, x.H, x.W, midp);
  G->creal = mid; G->cr = mid / 16;
  G->pooled = c->arena.alloc<float>(static_cast<size_t>(x.B) * 4 * midp);
  G->gates = c->arena.alloc<float>(static_cast<size_t>(x.B) * 4 * midp);
  G->w1 = c->arena.alloc<float>(static_cast<size_t>(G->cr) * mid); G->b1 = c->arena.alloc<float>(G->cr);
  G->w2 = c->arena.alloc<float>(static_cast<size_t>(mid) * G->cr); G->b2 = c->arena.alloc<float>(mid);
  Planes x2 = G->out;
  c->named.planes(pre + ".x1", x1);
  for (int k = 0; k < 4; ++k) c->named.planes(pre + ".s" + std::to_string(k), s[k]);
  c->named.planes(pre + ".x2", x2);
  const RGate* g = G.get();
  add_step(c->steps, 0, 0, "", [g](cudaStream_t st) {   // 4 x GAP + gate MLP + gated sum
    const int C = g->out.C, HW = g->out.H * g->out.W, B = g->out.B;
    for (int k = 0; k < 4; ++k)
      if (gap_launch(g->s[k].hi, g->s[k].lo, B, HW, C, g->pooled + static_cast<size_t>(k) * C, 4 * C, st)) return -1;
    if (gate_mlp_launch(g->pooled, B * 4, C, g->creal, g->cr, g->w1, g->b1, g->w2, g->b2, g->gates, st)) return -1;
    const __half* hi[4] = {g->s[0].hi, g->s[1].hi, g->s[2].hi, g->s[3].hi};
    const __half* lo[4] = {g->s[0].lo, g->s[1].lo, g->s[2].lo, g->s[3].lo};
    return gated_sum4_launch(hi, lo, g->gates, B, HW, C, g->out.hi, g->out.lo, st);
  }, 0, 0, 6);
  c->gates.push_back(std::move(G));
  Planes identity = x;
  if (cin != cout) {
    identity = c->planes(x.B, x.H, x.W, cout);
    add_conv(c, pre + ".downsample.conv.weight", pre + ".downsample.bn", "", x, cin, identity, cout, false, nullptr);
  }
  Planes out = c->planes(x.B, x.H, x.W, cout);
  add_conv(c, pre + ".conv3.conv.weight", pre + ".conv3.bn", "", x2, mid, out, cout, true, &identity);   // relu(x3 + identity)
  return out;
}

int build(b2_reid* c) {
  const int B = c->B;
  c->crops = c->arena.alloc<uint8_t>(static_cast<size_t>(B) * c->in_h * c->in_w * 3);
  const Planes c1 = add_stem(c, "conv1.conv.weight", "conv1.bn");   // osnet.py:307
  Planes x = add_maxpool(c, c1);                                       // :308
  const int chans[4] = {64, 256, 384, 512};
  for (int stage = 0; stage < 3; ++stage) {
    const std::string sn = "conv" + std::to_string(stage + 2);
    x = add_osblock(c, sn + ".0", x, chans[stage], chans[stage + 1]);
    c->named.planes(sn + ".0", x);
    x = add_osblock(c, sn + ".1", x, chans[stage + 1], chans[stage + 1]);
    c->named.planes(sn + ".1", x);
    if (stage < 2) {   // transition: Conv1x1 + AvgPool2d(2) (:375-381)
      Planes t = c->planes(B, x.H, x.W, x.C);
      add_conv(c, sn + ".2.0.conv.weight", sn + ".2.0.bn", "", x, x.C, t, x.C, true, nullptr);
      Planes q = c->planes(B, x.H / 2, x.W / 2, x.C);
      add_step(c->steps, 0, 0, "", [t, q](cudaStream_t st) {
        return avgpool2_launch(t.hi, t.lo, t.B, t.H, t.W, t.C, q.hi, q.lo, st);
      });
      c->named.planes(sn + ".t", t);
      x = q;
      c->named.planes(sn, x);
    }
  }
  Planes x5 = c->planes(B, x.H, x.W, 512);
  add_conv(c, "conv5.conv.weight", "conv5.bn", "", x, 512, x5, 512, true, nullptr);
  c->named.planes("conv5", x5);
  // global average pool -> fc + BN1d + ReLU (:428-431, fc built by _construct_fc_layer :386-405)
  const int Bp = (B + 127) / 128 * 128;
  c->gap_f32 = c->arena.alloc<float>(static_cast<size_t>(Bp) * 512);
  c->gap_planes = c->planes(1, 1, Bp, 512);
  const Planes gp = c->gap_planes;
  float* gap_f32 = c->gap_f32;
  add_step(c->steps, 0, 0, "", [x5, gp, gap_f32](cudaStream_t st) {
    if (gap_launch(x5.hi, x5.lo, x5.B, x5.H * x5.W, x5.C, gap_f32, x5.C, st)) return -1;
    return f32_to_planes(gap_f32, gp.hi, gp.lo, static_cast<size_t>(x5.B) * x5.C, st);
  }, 0, 0, 2);
  c->feats = c->arena.alloc<float>(static_cast<size_t>(Bp) * 512);
  Planes rows = c->gap_planes; rows.W = B;
  add_conv(c, "fc.0.weight", "fc.1", "fc.0.bias", rows, 512, Planes(), 512, true, nullptr, 1, 1, 0, c->feats, 512);
  return plan_convs(c->convs, c->split, c->num_sms);
}

// torchreid resnet101 (resnet.py:157-366): see the header comment.
int build_resnet101(b2_reid* c) {
  const int B = c->B;
  c->crops = c->arena.alloc<uint8_t>(static_cast<size_t>(B) * c->in_h * c->in_w * 3);
  const Planes c1 = add_stem(c, "conv1.weight", "bn1");                // conv1 7x7/2 pad 3 (:211-213)
  Planes x = add_maxpool(c, c1);                                       // maxpool 3/2 pad 1 (:216)
  const int blocks[4] = {3, 4, 23, 3}, planes[4] = {64, 128, 256, 512};
  for (int li = 0; li < 4; ++li) {
    const std::string ln = "layer" + std::to_string(li + 1);
    for (int bi = 0; bi < blocks[li]; ++bi) {
      const std::string pre = ln + "." + std::to_string(bi);
      const int stride = (bi == 0 && li > 0) ? 2 : 1;                 // _make_layer :246-290 (last_stride = 2)
      const int width = planes[li], cout = width * 4;
      if (stride == 2 && ((x.H | x.W) & 1)) {
        set_error("resnet101 reid: odd feature-map extent before a stride-2 layer");
        return -1;
      }
      const int ho = x.H / stride, wo = x.W / stride;
      Planes t1 = c->planes(B, x.H, x.W, width);
      add_conv(c, pre + ".conv1.weight", pre + ".bn1", "", x, x.C, t1, t1.C, true, nullptr);
      Planes t2 = c->planes(B, ho, wo, width);
      add_conv(c, pre + ".conv2.weight", pre + ".bn2", "", t1, t1.C, t2, t2.C, true, nullptr, 3, stride, 1);   // stride on the 3x3 (:126)
      Planes identity = x;
      if (bi == 0) {                                                   // downsample: conv1x1(stride) + BN (:262-268)
        identity = c->planes(B, ho, wo, cout);
        add_conv(c, pre + ".downsample.0.weight", pre + ".downsample.1", "", x, x.C, identity, cout, false, nullptr, 1, stride);
      }
      Planes out = c->planes(B, ho, wo, cout);
      add_conv(c, pre + ".conv3.weight", pre + ".bn3", "", t2, t2.C, out, cout, true, &identity);   // relu(bn3 + identity)
      x = out;
      c->named.planes(pre, x);
    }
    c->named.planes(ln, x);
  }
  const int Bp = (B + 127) / 128 * 128;
  c->feats = c->arena.alloc<float>(static_cast<size_t>(Bp) * c->feat_dim);
  float* feats = c->feats;
  add_step(c->steps, 0, 0, "", [x, feats](cudaStream_t st) {   // global_avgpool -> v (:355-359)
    return gap_launch(x.hi, x.lo, x.B, x.H * x.W, x.C, feats, x.C, st);
  });
  return plan_convs(c->convs, c->split, c->num_sms);
}

}  // namespace

extern "C" {

int b2_reid_create(b2_reid** out, int device, int batch, int precision) {
  return b2_reid_create_model(out, device, batch, precision, 0);
}

int b2_reid_create_model(b2_reid** out, int device, int batch, int precision, int model) {
  B2_CHECK(out && batch >= 1, "b2_reid_create: bad argument");
  *out = nullptr;
  B2_CHECK(model == 0 || model == 1, "b2_reid_create_model: model must be 0 (osnet_x1_0) or 1 (resnet101)");
  std::unique_ptr<b2_reid> c(new b2_reid());
  c->device = device; c->B = batch; c->split = precision == 1;
  c->model = model;
  if (model == 1) { c->in_h = 128; c->in_w = 256; c->feat_dim = 2048; }   // single_video_reid.py:410-415
  if (open_device(device, "b2_reid_create", &c->num_sms, &c->stream)) return -1;
  if ((model == 1 ? build_resnet101(c.get()) : build(c.get()))) { b2_reid_destroy(c.release()); return -1; }
  c->boxes = c->arena.alloc<int32_t>(static_cast<size_t>(batch) * 5);
  if (!c->boxes) { b2_reid_destroy(c.release()); return -1; }
  B2_CUDA(cudaDeviceSynchronize());
  *out = c.release();
  return 0;
}

void b2_reid_destroy(b2_reid* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  if (c->graph) cudaGraphExecDestroy(c->graph);
  if (c->stream) cudaStreamDestroy(c->stream);
  if (c->frames) cudaFree(c->frames);
  delete c;   // plans, then the arena's device memory
}

// state_dict of torchreid's osnet_x1_0 (names as model.state_dict(): "conv2.0.conv2b.1.conv1.weight", ...)
int b2_reid_load_weights(b2_reid* c, const char* const* names, const float* const* data, const int64_t* numel, int n) {
  B2_CHECK(c && names && data && numel, "b2_reid_load_weights: null argument");
  B2_CUDA(cudaSetDevice(c->device));
  const WeightSet ws(names, data, numel, n);
  for (auto& L : c->convs) {
    const int K = L->w.K, Cp = L->w.Cout_pad, co = L->d.Cout, ci = L->cin_real;
    std::vector<float> packed(static_cast<size_t>(Cp) * K, 0.f);
    std::vector<double> scale, shift;
    if (fold_bn(ws, L->bn, kTorchBn, 1e-5, co, scale, shift)) return -1;   // torch BatchNorm eps
    if (L->layout == kStem) {
      // torch OIHW [64,3,7,7] -> packed stem operand order (stem.cu): k = r*64 + s*12 + ry*6 + sx*3 + c
      const float* w = ws.get(L->name, 64 * 3 * 49);
      if (!w) return -1;
      for (int o = 0; o < 64; ++o)
        for (int r = 0; r < 4; ++r)
          for (int ch = 0; ch < 48; ++ch) {
            const int s4 = ch / 12, r12 = ch % 12, ry = r12 / 6, sx = (r12 % 6) / 3, cc = r12 % 3;
            const int rr = 2 * r + ry, ss = 2 * s4 + sx;
            if (rr >= 7 || ss >= 7) continue;
            packed[static_cast<size_t>(o) * K + r * 64 + ch] = static_cast<float>(w[((o * 3 + cc) * 7 + rr) * 7 + ss] * scale[o]);
          }
    } else if (L->layout == kOIHW) {
      // torch OIHW [co][ci][R][S] -> K-major [o][r][s][ci]
      const int R = L->d.R, S = L->d.S;
      const float* w = ws.get(L->name, static_cast<int64_t>(co) * ci * R * S);
      if (!w) return -1;
      for (int o = 0; o < co; ++o)
        for (int i = 0; i < ci; ++i)
          for (int r = 0; r < R; ++r)
            for (int q = 0; q < S; ++q)
              packed[static_cast<size_t>(o) * K + (static_cast<size_t>(r) * S + q) * ci + i] =
                  static_cast<float>(w[((static_cast<size_t>(o) * ci + i) * R + r) * S + q] * scale[o]);
    } else {
      const float* w = ws.get(L->name, static_cast<int64_t>(co) * ci);   // [O][I] (1x1 OIHW or Linear)
      if (!w) return -1;
      for (int o = 0; o < co; ++o)
        for (int i = 0; i < ci; ++i) packed[static_cast<size_t>(o) * K + i] = static_cast<float>(w[static_cast<size_t>(o) * ci + i] * scale[o]);
    }
    const float* b = nullptr;   // BN(Wx + b)
    if (!L->bias.empty() && !(b = ws.get(L->bias, co))) return -1;
    if (upload_conv(*L, packed, fold_bias(scale, shift, b, co, Cp), c->stream)) return -1;
  }
  for (auto& D : c->dws) {
    const int C = D->in.C, cr = D->creal;
    const float* w = ws.get(D->wname, static_cast<int64_t>(cr) * 9);   // [C,1,3,3]
    std::vector<double> scale, shift;
    if (!w || fold_bn(ws, D->bnname, kTorchBn, 1e-5, cr, scale, shift)) return -1;
    std::vector<float> pw(9 * C, 0.f), pb(C, 0.f);
    for (int ch = 0; ch < cr; ++ch) {
      for (int t = 0; t < 9; ++t) pw[t * C + ch] = static_cast<float>(w[ch * 9 + t] * scale[ch]);
      pb[ch] = static_cast<float>(shift[ch]);
    }
    B2_CUDA(cudaMemcpyAsync(D->w, pw.data(), pw.size() * 4, cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaMemcpyAsync(D->bias, pb.data(), pb.size() * 4, cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
  }
  for (auto& G : c->gates) {
    const int m = G->creal, r = G->cr;
    const float* w1 = ws.get(G->prefix + ".fc1.weight", static_cast<int64_t>(r) * m);
    const float* b1 = ws.get(G->prefix + ".fc1.bias", r);
    const float* w2 = ws.get(G->prefix + ".fc2.weight", static_cast<int64_t>(m) * r);
    const float* b2 = ws.get(G->prefix + ".fc2.bias", m);
    if (!w1 || !b1 || !w2 || !b2) return -1;
    B2_CUDA(cudaMemcpyAsync(G->w1, w1, sizeof(float) * r * m, cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaMemcpyAsync(G->b1, b1, sizeof(float) * r, cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaMemcpyAsync(G->w2, w2, sizeof(float) * m * r, cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaMemcpyAsync(G->b2, b2, sizeof(float) * m, cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaStreamSynchronize(c->stream));
  }
  c->loaded = true;
  return 0;
}

// crops: host RGB uint8 [n, in_h, in_w, 3] (already resized); the features go to `feats` (host, or device memory of the
// context's GPU when to_device)
static int reid_embed_impl(b2_reid* c, const uint8_t* crops_host, int n, float* feats, bool to_device) {
  B2_CHECK(c && crops_host && feats, "b2_reid_embed: null argument");
  B2_CHECK(n >= 1 && n <= c->B, "b2_reid_embed: batch larger than the context was created for");
  B2_CUDA(cudaSetDevice(c->device));
  B2_CHECK(c->loaded, "b2_reid_embed: weights not loaded");
  const size_t per = static_cast<size_t>(c->in_h) * c->in_w * 3;
  const cudaMemcpyKind out_kind = to_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  if (n < c->B) B2_CUDA(cudaMemsetAsync(c->crops + n * per, 0, (c->B - n) * per, c->stream));
  B2_CUDA(cudaMemcpyAsync(c->crops, crops_host, n * per, cudaMemcpyHostToDevice, c->stream));
  if (!c->graph && capture_graph(c->stream, [c] { return run_steps(c->steps, ~0u, c->stream); }, &c->graph)) return -1;
  B2_CUDA(cudaGraphLaunch(c->graph, c->stream));
  B2_CUDA(cudaMemcpyAsync(feats, c->feats, sizeof(float) * n * c->feat_dim, out_kind, c->stream));
  B2_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

int b2_reid_embed(b2_reid* c, const uint8_t* crops_host, int n, float* feats_host) {
  return reid_embed_impl(c, crops_host, n, feats_host, false);
}

// The features stay in HBM: `feats_dev` is device memory of the context's GPU (e.g. this camera's slice of the gallery
// buffer that the NCCL all-gather / the peer-memory pair cost of config 5 reads), so a gallery never crosses PCIe.
int b2_reid_embed_dev(b2_reid* c, const uint8_t* crops_host, int n, float* feats_dev) {
  return reid_embed_impl(c, crops_host, n, feats_dev, true);
}

// frames_host: uint8 BGR [nf][h][w][3]; boxes_host: [n][5] int32 (frame, x, y, w, h).  Every box is checked before anything
// is uploaded; the crop-resize kernel then fills the crop buffer the captured pass reads (rows n..B zeroed as above).
static int reid_embed_boxes_impl(b2_reid* c, const uint8_t* frames_host, int nf, int h, int w, const int32_t* boxes_host,
                                 int n, float* feats, bool to_device) {
  B2_CHECK(c && frames_host && boxes_host && feats, "b2_reid_embed_boxes: null argument");
  B2_CHECK(n >= 1 && n <= c->B, "b2_reid_embed_boxes: needs 1 <= n <= the batch the context was created for");
  B2_CHECK(nf >= 1 && h >= 1 && w >= 1, "b2_reid_embed_boxes: needs at least one frame of positive size");
  if (reid_boxes_check(boxes_host, n, nf, h, w, "b2_reid_embed_boxes")) return -1;
  B2_CUDA(cudaSetDevice(c->device));
  B2_CHECK(c->loaded, "b2_reid_embed_boxes: weights not loaded");
  const size_t per = static_cast<size_t>(c->in_h) * c->in_w * 3, frame_bytes = static_cast<size_t>(nf) * h * w * 3;
  if (frame_bytes > c->frames_cap) {
    B2_CUDA(cudaStreamSynchronize(c->stream));
    if (c->frames) B2_CUDA(cudaFree(c->frames));
    c->frames = nullptr;
    c->frames_cap = 0;
    B2_CUDA(cudaMalloc(&c->frames, frame_bytes));
    c->frames_cap = frame_bytes;
  }
  const cudaMemcpyKind out_kind = to_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  B2_CUDA(cudaMemcpyAsync(c->frames, frames_host, frame_bytes, cudaMemcpyHostToDevice, c->stream));
  B2_CUDA(cudaMemcpyAsync(c->boxes, boxes_host, sizeof(int32_t) * 5 * n, cudaMemcpyHostToDevice, c->stream));
  if (n < c->B) B2_CUDA(cudaMemsetAsync(c->crops + n * per, 0, (c->B - n) * per, c->stream));
  if (reid_crop_resize_launch(c->frames, h, w, c->boxes, n, c->crops, c->in_h, c->in_w, c->stream)) return -1;
  if (!c->graph && capture_graph(c->stream, [c] { return run_steps(c->steps, ~0u, c->stream); }, &c->graph)) return -1;
  B2_CUDA(cudaGraphLaunch(c->graph, c->stream));
  B2_CUDA(cudaMemcpyAsync(feats, c->feats, sizeof(float) * n * c->feat_dim, out_kind, c->stream));
  B2_CUDA(cudaStreamSynchronize(c->stream));
  return 0;
}

int b2_reid_embed_boxes(b2_reid* c, const uint8_t* frames_host, int nf, int h, int w, const int32_t* boxes_host, int n,
                        float* feats_host) {
  return reid_embed_boxes_impl(c, frames_host, nf, h, w, boxes_host, n, feats_host, false);
}

int b2_reid_embed_boxes_dev(b2_reid* c, const uint8_t* frames_host, int nf, int h, int w, const int32_t* boxes_host, int n,
                            float* feats_dev) {
  return reid_embed_boxes_impl(c, frames_host, nf, h, w, boxes_host, n, feats_dev, true);
}

int b2_reid_feat_dim(b2_reid* c) { return c ? c->feat_dim : -1; }

// Stage-addressable activation of the last pass as fp32 NHWC (names: "stem_u", "conv1", "maxpool", "conv2.0", "conv2.0.x1",
// "conv2.0.s0".."s3", "conv2.0.x2", "conv2.1", "conv2", ..., "conv5").
int b2_reid_get_activation(b2_reid* c, const char* name, float* dst, int64_t capacity, int64_t shape[4]) {
  B2_CHECK(c && name && dst && shape, "b2_reid_get_activation: null argument");
  B2_CUDA(cudaSetDevice(c->device));
  return stage_get(c->named, name, c->stream, dst, capacity, shape, "b2_reid_get_activation");
}

int b2_reid_num_launches(b2_reid* c) { return c ? total_launches(c->steps) : -1; }

}  // extern "C"
