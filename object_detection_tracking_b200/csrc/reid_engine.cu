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
//
// resnet101 is one row of the ResNet family table (kResnet, b2_reid_create_named): resnet18 / resnet34 (BasicBlock,
// resnet.py:52-102), resnet50 / resnet152, resnext50_32x4d / resnext101_32x8d (conv2 grouped 32 ways, on the conv kernel's
// block-diagonal 64-channel windows), resnet50_fc512 (last stride 1, then fc 2048 -> 512 + BN1d + ReLU), resnet50_ibn_a
// (resnet_ibn_a.py: bn1 of layer1-3 = IN of the first planes/2 channels beside BN of the rest, instnorm_split_launch) and
// resnet50_ibn_b (resnet_ibn_b.py: IN stem, IN after the residual of layer1.2 and layer2.3).
//
// The rest of torchreid's OSNet family (models 2-6) builds from the same blocks through a per-model table (kOsnet):
// the x0.75 / x0.5 / x0.25 widths (osnet.py:537-579) carry channel counts that are not multiples of 64 as zero-padded
// planes, and osnet_ibn_x1_0 (osnet.py:582-598) / osnet_ain_x1_0 (osnet_ain.py:524-541) add InstanceNorm2d steps
// (instnorm_launch, reid.cu) on the stem and on the blocks the table marks.
#include <math.h>
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

// InstanceNorm2d(affine) of x, then + res (when res.hi) and ReLU, into y; with c_norm, IBN-a's split (channels
// [0, c_norm) normalised, the rest passed through)
struct RIn {
  std::string prefix;      // "...IN" / "conv1.bn": .weight / .bias in the state_dict
  Planes x, res, y;
  float *gamma = nullptr, *beta = nullptr;   // [C], zero on padded channels
  int creal = 0;           // channels with a gamma / beta
  int c_norm = 0;          // 0: every channel (instnorm_launch); else instnorm_split_launch
  bool relu = true;
};

// ConvLayer::layout: how the torch weight is packed
// [O][I] (1x1 OIHW or Linear), packed 7x7 stem, RxS conv OIHW, grouped RxS conv OIHW [O][I/groups][R][S]
enum { kOI = 0, kStem = 1, kOIHW = 2, kGroupedOIHW = 3 };

// OSNet block kinds: OSBlock; OSBlock with IN after the residual add (osnet.py:270-276, IN=True); OSBlockINin, IN on
// the bare conv3 inside the residual (osnet_ain.py:263-295)
enum { kPlainBlock = 0, kIbnBlock = 1, kINinBlock = 2 };

struct OsnetSpec {
  const char* name;
  int ch[4];                 // channels (osnet.py:310-334): stem, conv2, conv3, conv4 outputs
  bool stem_in;              // conv1 is conv -> IN -> ReLU
  int kind[3][2];            // block kind of convN.0 / convN.1
  bool ain_names;            // osnet_ain.py's module names: convN.M.conv2.{t}.layers.{j} streams, poolN.0 transitions
};

const OsnetSpec kOsnet[] = {
    {"osnet_x1_0", {64, 256, 384, 512}, false, {{0, 0}, {0, 0}, {0, 0}}, false},
    {"osnet_x0_75", {48, 192, 288, 384}, false, {{0, 0}, {0, 0}, {0, 0}}, false},
    {"osnet_x0_5", {32, 128, 192, 256}, false, {{0, 0}, {0, 0}, {0, 0}}, false},
    {"osnet_x0_25", {16, 64, 96, 128}, false, {{0, 0}, {0, 0}, {0, 0}}, false},
    {"osnet_ibn_x1_0", {64, 256, 384, 512}, true, {{1, 1}, {0, 0}, {0, 0}}, false},
    {"osnet_ain_x1_0", {64, 256, 384, 512}, true, {{2, 2}, {0, 2}, {2, 0}}, true},
};

// torchreid's ResNet family (resnet.py:157-530, resnet_ibn_a.py:131-289, resnet_ibn_b.py:114-274)
enum { kBasic = 0, kBottleneck = 1 };
enum { kNoIbn = 0, kIbnA = 1, kIbnB = 2 };

struct ResnetSpec {
  const char* name;
  int block;               // kBasic (expansion 1) or kBottleneck (expansion 4)
  int layers[4];           // blocks of layer1..4
  int groups, width;       // conv2's groups and width per group: a Bottleneck's conv2 is planes * width / 64 * groups wide
  int last_stride;         // layer4's stride
  int fc;                  // fc_dims = [fc]: Linear + BatchNorm1d + ReLU after the pool; 0 = none
  int ibn;                 // kIbnA: bn1 of layer1-3 is IBN; kIbnB: IN stem, IN after layer1 / layer2's last residual
  bool person;             // built at 256x128 (torchreid's default) as well as at 128x256
};

const ResnetSpec kResnet[] = {
    {"resnet101", kBottleneck, {3, 4, 23, 3}, 1, 64, 2, 0, kNoIbn, false},
    {"resnet18", kBasic, {2, 2, 2, 2}, 1, 64, 2, 0, kNoIbn, true},
    {"resnet34", kBasic, {3, 4, 6, 3}, 1, 64, 2, 0, kNoIbn, true},
    {"resnet50", kBottleneck, {3, 4, 6, 3}, 1, 64, 2, 0, kNoIbn, true},
    {"resnet152", kBottleneck, {3, 8, 36, 3}, 1, 64, 2, 0, kNoIbn, true},
    {"resnext50_32x4d", kBottleneck, {3, 4, 6, 3}, 32, 4, 2, 0, kNoIbn, true},
    {"resnext101_32x8d", kBottleneck, {3, 4, 23, 3}, 32, 8, 2, 0, kNoIbn, true},
    {"resnet50_fc512", kBottleneck, {3, 4, 6, 3}, 1, 64, 1, 512, kNoIbn, true},
    {"resnet50_ibn_a", kBottleneck, {3, 4, 6, 3}, 1, 64, 2, 0, kIbnA, true},
    {"resnet50_ibn_b", kBottleneck, {3, 4, 6, 3}, 1, 64, 2, 0, kIbnB, true},
};

}  // namespace

struct b2_reid {
  Arena arena;                       // first member: freed after everything that refers to it
  int device = 0, num_sms = 132, B = 0;
  const OsnetSpec* osnet = nullptr;  // the model: a row of kOsnet or of kResnet
  const ResnetSpec* resnet = nullptr;
  int in_h = 256, in_w = 128;        // crop size (h, w) the extractor resizes to
  int feat_dim = 512;
  bool split = true;
  cudaStream_t stream = nullptr;
  std::vector<std::unique_ptr<ConvLayer>> convs;
  std::vector<std::unique_ptr<RDw>> dws;
  std::vector<std::unique_ptr<RGate>> gates;
  std::vector<std::unique_ptr<RIn>> ins;
  std::map<const ConvLayer*, int> bn_from;   // IBN-a conv1: its BN covers output channels [bn_from, Cout) only
  std::vector<Step> steps;
  StageMap named;                    // stage-addressable activations (parity tests)
  uint8_t* crops = nullptr;          // [B][in_h][in_w][3] RGB, the stem pack's input
  uint8_t* frames = nullptr;         // b2_reid_embed_boxes: uploaded frames, grow-only (cudaMalloc, freed on destroy)
  size_t frames_cap = 0;
  int32_t* boxes = nullptr;          // [B][5] box table of the last b2_reid_embed_boxes call
  Planes stem_u, gap_planes;
  float* gap_f32 = nullptr;
  float* feats = nullptr;      // [Bpad][feat_dim]
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
                    int pad = 0, float* out_f32 = nullptr, int ldc32 = 0, int groups = 1) {
  ConvDesc d;
  d.R = d.S = k; d.stride = stride; d.groups = groups;
  d.pad_t = d.pad_l = pad;
  // stride 2 on even extents: the last window ends one row / column before torch's bottom / right padding, so
  // (pad, pad - 1) is the same convolution -- and exactly the geometry the detector's strided layers use
  // (nn.py:487-492 3x3 with pads (1,0); :555-560 1x1 with the last row / column dropped).
  d.pad_b = d.pad_r = stride == 2 ? pad - 1 : pad;
  d.Cout = cout_real; d.relu = relu ? 1 : 0;
  std::unique_ptr<ConvLayer> L = make_conv(c->arena, c->split, wname, d, in, out, res, out_f32, ldc32);
  L->bn = bn; L->bias = bias; L->cin_real = cin_real;
  L->layout = groups > 1 ? kGroupedOIHW : (k != 1 || stride != 1) ? kOIHW : kOI;
  ConvLayer* raw = L.get();
  add_conv_step(c->steps, 0, raw);
  c->convs.push_back(std::move(L));
  return raw;
}

// conv1 7x7/2 pad 3 through the packed-operand trick of stem.cu: a 4x1 VALID conv over the packed operand, with `cout`
// outputs padded to 64; BN + ReLU in the epilogue, or (bn empty, relu false) the bare conv an InstanceNorm follows
Planes add_stem(b2_reid* c, const std::string& wname, const std::string& bn, int cout = 64, bool relu = true) {
  const int B = c->B, h1 = (c->in_h + 6 - 7) / 2 + 1, w1 = (c->in_w + 6 - 7) / 2 + 1;
  c->stem_u = c->planes(B, h1 + 3, w1, 64);
  const Planes u = c->stem_u;
  add_step(c->steps, 0, 0, "", [c, u](cudaStream_t st) {
    return stem_pack_launch(c->crops, c->B, c->in_h, c->in_w, u.hi, u.lo, u.H, u.W, st);
  });
  Planes c1 = c->planes(B, h1, w1, pad64(cout));
  ConvDesc d;
  d.R = 4; d.S = 1; d.Cout = cout; d.relu = relu ? 1 : 0;
  std::unique_ptr<ConvLayer> L = make_conv(c->arena, c->split, wname, d, c->stem_u, c1);
  L->bn = bn; L->cin_real = 64; L->layout = kStem;
  add_conv_step(c->steps, 0, L.get());
  c->convs.push_back(std::move(L));
  c->named.planes("stem_u", c->stem_u);
  c->named.planes("conv1", c1);
  return c1;
}

// InstanceNorm2d(creal, affine=True) `prefix` of x, then + res (may be null) and ReLU, into new planes.  With c_norm:
// IBN-a's split, the IN of channels [0, c_norm) only (creal == c_norm), the others passed through to the ReLU.
Planes add_instnorm(b2_reid* c, const std::string& prefix, const Planes& x, const Planes* res, int creal, int c_norm = 0) {
  std::unique_ptr<RIn> N(new RIn());
  N->prefix = prefix; N->x = x; N->creal = creal; N->c_norm = c_norm;
  if (res) N->res = *res;
  N->y = c->planes(x.B, x.H, x.W, x.C);
  N->gamma = c->arena.alloc<float>(x.C); N->beta = c->arena.alloc<float>(x.C);
  const RIn* n = N.get();
  add_step(c->steps, 0, 0, prefix, [n](cudaStream_t st) {
    if (n->c_norm)
      return instnorm_split_launch(n->x.hi, n->x.lo, n->x.B, n->x.H * n->x.W, n->x.C, n->c_norm, n->gamma, n->beta, n->y.hi,
                                   n->y.lo, st);
    return instnorm_launch(n->x.hi, n->x.lo, n->res.hi, n->res.lo, n->x.B, n->x.H * n->x.W, n->x.C, n->gamma, n->beta,
                           n->relu ? 1 : 0, n->y.hi, n->y.lo, st);
  });
  c->ins.push_back(std::move(N));
  return n->y;
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

// OSBlock (osnet.py:223-276, osnet_ain.py:230-260) or OSBlockINin (osnet_ain.py:263-295) by `kind`; cin / cout are the
// model's channel counts, the planes carry them padded to 64
Planes add_osblock(b2_reid* c, const std::string& pre, const Planes& x, int cin, int cout, int kind = kPlainBlock,
                   bool ain_names = false) {
  const int mid = cout / 4, midp = pad64(mid);
  Planes x1 = c->planes(x.B, x.H, x.W, midp);
  add_conv(c, pre + ".conv1.conv.weight", pre + ".conv1.bn", "", x, cin, x1, mid, true, nullptr);
  Planes s[4];
  const char* names[4] = {".conv2a", ".conv2b", ".conv2c", ".conv2d"};
  for (int k = 0; k < 4; ++k) {
    Planes t = x1;
    if (ain_names)   // LightConvStream of depth k + 1 (osnet_ain.py:148-163)
      for (int j = 0; j <= k; ++j) t = add_light(c, pre + ".conv2." + std::to_string(k) + ".layers." + std::to_string(j), t, mid);
    else if (k == 0) t = add_light(c, pre + names[k], t, mid);
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
    identity = c->planes(x.B, x.H, x.W, pad64(cout));
    add_conv(c, pre + ".downsample.conv.weight", pre + ".downsample.bn", "", x, cin, identity, cout, false, nullptr);
  }
  Planes out = c->planes(x.B, x.H, x.W, pad64(cout));
  if (kind == kPlainBlock) {
    add_conv(c, pre + ".conv3.conv.weight", pre + ".conv3.bn", "", x2, mid, out, cout, true, &identity);   // relu(x3 + identity)
    return out;
  }
  if (kind == kIbnBlock) {   // relu(IN(x3 + identity))
    add_conv(c, pre + ".conv3.conv.weight", pre + ".conv3.bn", "", x2, mid, out, cout, false, &identity);
    c->named.planes(pre + ".pre_in", out);
    return add_instnorm(c, pre + ".IN", out, nullptr, cout);
  }
  // relu(IN(conv3(x2)) + identity), conv3 without BN or bias
  add_conv(c, pre + ".conv3.conv.weight", "", "", x2, mid, out, cout, false, nullptr);
  c->named.planes(pre + ".pre_in", out);
  return add_instnorm(c, pre + ".IN", out, &identity, cout);
}

// global average pool of x -> fp32 rows -> fc.0 (Linear cin_real -> dim) + fc.1 (BatchNorm1d) + ReLU into c->feats
// (osnet.py:386-405, 428-431; resnet.py:292-320, 353-362)
void add_gap_fc(b2_reid* c, const Planes& x5, int cin_real, int dim) {
  const int B = c->B, Bp = (B + 127) / 128 * 128;
  c->gap_f32 = c->arena.alloc<float>(static_cast<size_t>(Bp) * x5.C);
  c->gap_planes = c->planes(1, 1, Bp, x5.C);
  const Planes gp = c->gap_planes;
  float* gap_f32 = c->gap_f32;
  add_step(c->steps, 0, 0, "", [x5, gp, gap_f32](cudaStream_t st) {
    if (gap_launch(x5.hi, x5.lo, x5.B, x5.H * x5.W, x5.C, gap_f32, x5.C, st)) return -1;
    return f32_to_planes(gap_f32, gp.hi, gp.lo, static_cast<size_t>(x5.B) * x5.C, st);
  }, 0, 0, 2);
  c->feats = c->arena.alloc<float>(static_cast<size_t>(Bp) * dim);
  Planes rows = c->gap_planes; rows.W = B;
  add_conv(c, "fc.0.weight", "fc.1", "fc.0.bias", rows, cin_real, Planes(), dim, true, nullptr, 1, 1, 0, c->feats, dim);
}

int build_osnet(b2_reid* c) {
  const int B = c->B;
  const OsnetSpec& m = *c->osnet;
  c->crops = c->arena.alloc<uint8_t>(static_cast<size_t>(B) * c->in_h * c->in_w * 3);
  Planes c1;
  if (m.stem_in) {   // ConvLayer(IN=True): conv -> InstanceNorm2d -> ReLU (osnet.py:28-61)
    const Planes pre = add_stem(c, "conv1.conv.weight", "", m.ch[0], false);
    c1 = add_instnorm(c, "conv1.bn", pre, nullptr, m.ch[0]);
    c->named.planes("conv1.pre_in", pre);
    c->named.planes("conv1", c1);
  } else {
    c1 = add_stem(c, "conv1.conv.weight", "conv1.bn", m.ch[0]);     // osnet.py:307
  }
  Planes x = add_maxpool(c, c1);                                       // :308
  const int* chans = m.ch;
  for (int stage = 0; stage < 3; ++stage) {
    const std::string sn = "conv" + std::to_string(stage + 2);
    x = add_osblock(c, sn + ".0", x, chans[stage], chans[stage + 1], m.kind[stage][0], m.ain_names);
    c->named.planes(sn + ".0", x);
    x = add_osblock(c, sn + ".1", x, chans[stage + 1], chans[stage + 1], m.kind[stage][1], m.ain_names);
    c->named.planes(sn + ".1", x);
    if (stage < 2) {   // transition: Conv1x1 + AvgPool2d(2) (:375-381; osnet_ain.py:336-344 names it poolN.0)
      const std::string tn = m.ain_names ? "pool" + std::to_string(stage + 2) + ".0" : sn + ".2.0";
      const int cr = chans[stage + 1];
      Planes t = c->planes(B, x.H, x.W, x.C);
      add_conv(c, tn + ".conv.weight", tn + ".bn", "", x, cr, t, cr, true, nullptr);
      Planes q = c->planes(B, x.H / 2, x.W / 2, x.C);
      add_step(c->steps, 0, 0, "", [t, q](cudaStream_t st) {
        return avgpool2_launch(t.hi, t.lo, t.B, t.H, t.W, t.C, q.hi, q.lo, st);
      });
      c->named.planes(sn + ".t", t);
      x = q;
      c->named.planes(sn, x);
    }
  }
  const int c5 = chans[3];   // conv5 and the fc input are channels[3] wide (osnet.py:334-339); the feature stays 512
  Planes x5 = c->planes(B, x.H, x.W, pad64(c5));
  add_conv(c, "conv5.conv.weight", "conv5.bn", "", x, c5, x5, c5, true, nullptr);
  c->named.planes("conv5", x5);
  add_gap_fc(c, x5, c5, 512);   // global average pool -> fc + BN1d + ReLU
  return plan_convs(c->convs, c->split, c->num_sms);
}

// torchreid's ResNet family by its kResnet row (resnet.py:157-366; see the header comment).  Stage names: "conv1",
// "maxpool", "layerN.M", "layerN", and for each InstanceNorm "<stage>.pre_in" for its input ("conv1.pre_in",
// "layer1.2.pre_in"; IBN-a: "layerN.M.bn1.pre_in" and "layerN.M.bn1").
int build_resnet(b2_reid* c) {
  const ResnetSpec& m = *c->resnet;
  const int B = c->B;
  c->crops = c->arena.alloc<uint8_t>(static_cast<size_t>(B) * c->in_h * c->in_w * 3);
  Planes c1;
  if (m.ibn == kIbnB) {   // bn1 = InstanceNorm2d(64, affine) (resnet_ibn_b.py:142)
    const Planes pre = add_stem(c, "conv1.weight", "", 64, false);
    c1 = add_instnorm(c, "bn1", pre, nullptr, 64);
    c->named.planes("conv1.pre_in", pre);
    c->named.planes("conv1", c1);
  } else {
    c1 = add_stem(c, "conv1.weight", "bn1");                         // conv1 7x7/2 pad 3 (:211-213)
  }
  Planes x = add_maxpool(c, c1);                                     // maxpool 3/2 pad 1 (:216)
  int cin = 64;
  for (int li = 0; li < 4; ++li) {
    const std::string ln = "layer" + std::to_string(li + 1);
    const int planes = 64 << li;
    const int cout = m.block == kBasic ? planes : planes * 4;
    const int width = m.block == kBasic ? planes : planes * m.width / 64 * m.groups;   // Bottleneck :122
    for (int bi = 0; bi < m.layers[li]; ++bi) {
      const std::string pre = ln + "." + std::to_string(bi);
      const int stride = bi > 0 || li == 0 ? 1 : li == 3 ? m.last_stride : 2;       // _make_layer :257-290
      if (stride == 2 && ((x.H | x.W) & 1)) {
        set_error(std::string(m.name) + " reid: odd feature-map extent before a stride-2 layer");
        return -1;
      }
      const int ho = x.H / stride, wo = x.W / stride;
      const bool down = bi == 0 && (stride != 1 || cin != cout);    // downsample: conv1x1(stride) + BN (:264-268)
      auto add_downsample = [&]() {
        Planes identity = x;
        if (down) {
          identity = c->planes(B, ho, wo, cout);
          add_conv(c, pre + ".downsample.0.weight", pre + ".downsample.1", "", x, x.C, identity, cout, false, nullptr, 1,
                   stride);
        }
        return identity;
      };
      Planes out = c->planes(B, ho, wo, cout);
      if (m.block == kBasic) {   // BasicBlock (:52-102): 3x3 carrying the stride, 3x3 with the residual
        Planes t1 = c->planes(B, ho, wo, width);
        add_conv(c, pre + ".conv1.weight", pre + ".bn1", "", x, x.C, t1, width, true, nullptr, 3, stride, 1);
        const Planes identity = add_downsample();
        add_conv(c, pre + ".conv2.weight", pre + ".bn2", "", t1, width, out, cout, true, &identity, 3, 1, 1);
      } else {
        Planes t1 = c->planes(B, x.H, x.W, width);
        const bool ibn_a = m.ibn == kIbnA && li < 3;                 // resnet_ibn_a.py:198-200
        ConvLayer* conv1 = add_conv(c, pre + ".conv1.weight", pre + (ibn_a ? ".bn1.BN" : ".bn1"), "", x, x.C, t1, width,
                                    !ibn_a, nullptr);
        if (ibn_a) {   // IBN (resnet_ibn_a.py:63-79): conv1's epilogue ran BN on channels [width / 2, width) only
          c->bn_from[conv1] = width / 2;
          c->named.planes(pre + ".bn1.pre_in", t1);
          t1 = add_instnorm(c, pre + ".bn1.IN", t1, nullptr, width / 2, width / 2);
          c->named.planes(pre + ".bn1", t1);
        }
        Planes t2 = c->planes(B, ho, wo, width);
        add_conv(c, pre + ".conv2.weight", pre + ".bn2", "", t1, t1.C, t2, t2.C, true, nullptr, 3, stride, 1, nullptr, 0,
                 m.groups);                                          // stride on the 3x3 (:126)
        const Planes identity = add_downsample();
        // resnet_ibn_b.py:106-109, 184-189: relu(IN(bn3 + identity)) in the last block of layer1 and layer2
        const bool ibn_b = m.ibn == kIbnB && li < 2 && bi == m.layers[li] - 1;
        add_conv(c, pre + ".conv3.weight", pre + ".bn3", "", t2, t2.C, out, cout, !ibn_b, &identity);   // relu(bn3 + identity)
        if (ibn_b) {
          c->named.planes(pre + ".pre_in", out);
          out = add_instnorm(c, pre + ".IN", out, nullptr, cout);
        }
      }
      x = out;
      cin = cout;
      c->named.planes(pre, x);
    }
    c->named.planes(ln, x);
  }
  if (m.fc) {
    add_gap_fc(c, x, cin, m.fc);
  } else {
    const int Bp = (B + 127) / 128 * 128;
    c->feats = c->arena.alloc<float>(static_cast<size_t>(Bp) * c->feat_dim);
    float* feats = c->feats;
    add_step(c->steps, 0, 0, "", [x, feats](cudaStream_t st) {   // global_avgpool -> v (:355-359)
      return gap_launch(x.hi, x.lo, x.B, x.H * x.W, x.C, feats, x.C, st);
    });
  }
  return plan_convs(c->convs, c->split, c->num_sms);
}

// "name at HxW, ..." for every model and crop size b2_reid_create_named builds
std::string built_models() {
  std::string s;
  for (const OsnetSpec& m : kOsnet) s += std::string(s.empty() ? "" : ", ") + m.name + " at 256x128";
  for (const ResnetSpec& m : kResnet) s += std::string(", ") + m.name + (m.person ? " at 256x128 or 128x256" : " at 128x256");
  return s;
}

}  // namespace

extern "C" {

int b2_reid_create(b2_reid** out, int device, int batch, int precision) {
  return b2_reid_create_model(out, device, batch, precision, 0);
}

int b2_reid_create_model(b2_reid** out, int device, int batch, int precision, int model) {
  B2_CHECK(out && batch >= 1, "b2_reid_create: bad argument");
  *out = nullptr;
  B2_CHECK(model >= 0 && model <= 6,
           "b2_reid_create_model: model must be 0 (osnet_x1_0), 1 (resnet101), 2 (osnet_x0_75), 3 (osnet_x0_5), "
           "4 (osnet_x0_25), 5 (osnet_ibn_x1_0) or 6 (osnet_ain_x1_0)");
  static const char* const kIds[7] = {"osnet_x1_0", "resnet101", "osnet_x0_75", "osnet_x0_5", "osnet_x0_25",
                                      "osnet_ibn_x1_0", "osnet_ain_x1_0"};
  const bool vehicle = model == 1;   // single_video_reid.py:410-415
  return b2_reid_create_named(out, device, batch, precision, kIds[model], vehicle ? 128 : 256, vehicle ? 256 : 128);
}

int b2_reid_create_named(b2_reid** out, int device, int batch, int precision, const char* model, int in_h, int in_w) {
  B2_CHECK(out && batch >= 1 && model, "b2_reid_create_named: bad argument");
  *out = nullptr;
  std::unique_ptr<b2_reid> c(new b2_reid());
  for (const OsnetSpec& m : kOsnet)
    if (!strcmp(m.name, model)) c->osnet = &m;
  for (const ResnetSpec& m : kResnet)
    if (!strcmp(m.name, model)) c->resnet = &m;
  const bool person = in_h == 256 && in_w == 128, vehicle = in_h == 128 && in_w == 256;
  B2_CHECK(c->osnet ? person : c->resnet && (vehicle || (person && c->resnet->person)),
           std::string("b2_reid_create_named: ") + model + " at " + std::to_string(in_h) + "x" + std::to_string(in_w) +
               " is not built; the models are " + built_models());
  c->device = device; c->B = batch; c->split = precision == 1;
  c->in_h = in_h; c->in_w = in_w;
  if (c->resnet) c->feat_dim = c->resnet->fc ? c->resnet->fc : c->resnet->block == kBasic ? 512 : 2048;
  if (open_device(device, "b2_reid_create", &c->num_sms, &c->stream)) return -1;
  if ((c->resnet ? build_resnet(c.get()) : build_osnet(c.get()))) { b2_reid_destroy(c.release()); return -1; }
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

// state_dict of the context's torchreid model (names as model.state_dict(): "conv2.0.conv2b.1.conv1.weight", ...)
int b2_reid_load_weights(b2_reid* c, const char* const* names, const float* const* data, const int64_t* numel, int n) {
  B2_CHECK(c && names && data && numel, "b2_reid_load_weights: null argument");
  B2_CUDA(cudaSetDevice(c->device));
  const WeightSet ws(names, data, numel, n);
  for (auto& L : c->convs) {
    const int K = L->w.K, Cp = L->w.Cout_pad, co = L->d.Cout, ci = L->cin_real;
    std::vector<float> packed(static_cast<size_t>(Cp) * K, 0.f);
    std::vector<double> scale, shift;
    const auto split = c->bn_from.find(L.get());   // IBN-a: channels [0, c_bn) leave conv1 raw for the InstanceNorm
    const int c_bn = split == c->bn_from.end() ? 0 : split->second;
    if (fold_bn(ws, L->bn, kTorchBn, 1e-5, co - c_bn, scale, shift)) return -1;   // torch BatchNorm eps
    scale.insert(scale.begin(), c_bn, 1.0);
    shift.insert(shift.begin(), c_bn, 0.0);
    if (L->layout == kStem) {
      // torch OIHW [co,3,7,7] -> packed stem operand order (stem.cu): k = r*64 + s*12 + ry*6 + sx*3 + c
      const float* w = ws.get(L->name, static_cast<int64_t>(co) * 3 * 49);
      if (!w) return -1;
      for (int o = 0; o < co; ++o)
        for (int r = 0; r < 4; ++r)
          for (int ch = 0; ch < 48; ++ch) {
            const int s4 = ch / 12, r12 = ch % 12, ry = r12 / 6, sx = (r12 % 6) / 3, cc = r12 % 3;
            const int rr = 2 * r + ry, ss = 2 * s4 + sx;
            if (rr >= 7 || ss >= 7) continue;
            packed[static_cast<size_t>(o) * K + r * 64 + ch] = static_cast<float>(w[((o * 3 + cc) * 7 + rr) * 7 + ss] * scale[o]);
          }
    } else if (L->layout == kGroupedOIHW) {
      // torch OIHW [co][ci/groups][R][S] -> HWIO [r*S+s][ci/groups][co] -> the conv kernel's block-diagonal windows
      const int RS = L->d.R * L->d.S, cg = ci / L->d.groups;
      const float* w = ws.get(L->name, static_cast<int64_t>(co) * cg * RS);
      if (!w) return -1;
      std::vector<float> hwio(static_cast<size_t>(RS) * cg * co);
      for (int o = 0; o < co; ++o)
        for (int i = 0; i < cg; ++i)
          for (int t = 0; t < RS; ++t)
            hwio[(static_cast<size_t>(t) * cg + i) * co + o] = w[(static_cast<size_t>(o) * cg + i) * RS + t];
      pack_grouped(hwio.data(), RS, ci, co, L->d.groups, scale.data(), K, packed);
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
  for (auto& N : c->ins) {   // InstanceNorm2d affine: weight / bias only (track_running_stats=False)
    const int C = N->x.C, cr = N->creal;
    const float* g = ws.get(N->prefix + ".weight", cr);
    const float* b = ws.get(N->prefix + ".bias", cr);
    if (!g || !b) return -1;
    std::vector<float> pg(C, 0.f), pb(C, 0.f);
    for (int ch = 0; ch < cr; ++ch) {
      pg[ch] = g[ch];
      pb[ch] = b[ch];
    }
    B2_CUDA(cudaMemcpyAsync(N->gamma, pg.data(), sizeof(float) * C, cudaMemcpyHostToDevice, c->stream));
    B2_CUDA(cudaMemcpyAsync(N->beta, pb.data(), sizeof(float) * C, cudaMemcpyHostToDevice, c->stream));
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
