// The detector's launch plan and the builders that append to it: conv layers, GroupNorm, squeeze-excite, relation and
// deformable steps and the ResNet blocks made of them, plus the loader that fills their weights from a checkpoint.  The
// detector engine (engine.cu) builds its whole plan with them; the single-op entry points (ops.cu) build one-block plans
// with the same builders, so that their tests check the code the detector runs.
#pragma once
#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "engine_core.h"
#include "kernels.h"

namespace b2 {

// One GroupNorm of the plan (use_gn backbone / FPN, conv box head): normalises a conv output in place.
struct GnOp {
  std::string name;        // reference variable scope, e.g. "group1/block0/conv1/gn", "fpn/gn_c2", "fastrcnn/gn0"
  GnParams p;              // full-batch launch (its gamma / beta are loaded with the weights)
};

// The squeeze-excite of one SE-ResNet bottleneck (use_se): the dense weights "<name>/fc1/{W,b}" and "<name>/fc2/{W,b}".
struct SeOp {
  std::string name;        // block scope, e.g. "group1/block0"
  int C = 0, nr = 0;       // 4 * ch_out gated channels, ch_out / 4 hidden units
  float *w1 = nullptr, *b1 = nullptr, *w2 = nullptr, *b2 = nullptr;   // [C][nr], [nr], [nr][C], [C]
  float* gate = nullptr;   // [B][C], written by the excite step
};

// The geometry weights of one relation module (add_relation_nn): "<scope>/geo_emb/{W,b}", "<scope>/geo_conv/{W,b}".
struct RelOp {
  std::string name;        // module scope, "fastrcnn/RM_r1" or "fastrcnn/RM_r2"
  float* geo = nullptr;    // kRelGeoWeights (relation_upload_geo)
};

// Packing of a checkpoint weight into the [Cout_pad][K] operand (ConvLayer::layout).
enum Layout {
  kHwio = 0,     // conv HWIO
  kFc6 = 1,      // dense over the NCHW flatten of [7][7][C] ROI features
  kDense = 2,
  kRpnOut = 3,   // rpn/{class,box} fused along N
  kHeadOut = 4,  // fastrcnn/outputs/{class,box} fused along N
  kStem = 5,     // 7x7 stem re-indexed for the packed operand
  kDeconv = 6,   // mask-head transposed conv 2x2/2 as a 1x1 conv onto 4 taps x C outputs
  kGrouped = 7,  // grouped conv HWIO [R][S][Cin/groups][Cout] (pack_grouped)
  kRelQK = 8,    // relation module: <scope>/query_linear/W | <scope>/key_linear/W fused along N (relation_pack_qk)
  kRuntime = 9,  // relation module P.V: the weights are the image's V^T, written by the attention step every pass
  kShared = 10,  // another layer's packed weights (add_conv_shared): nothing of its own to load
  kSoClass = 11, // small-object classification: fastrcnn/small_objects/small_object_classification_c{i+1}/{W,b}, [D, 2]
                 // each, as columns 2i, 2i + 1
};

// The checkpoint's per-channel affine of a conv output, applied in the epilogue: none, the folded BatchNorm "<name>/bn"
// or the bias "<name>/b".
enum ConvAffine { kNoAffine, kBatchNorm, kBias };

// Step kinds as b2_step_info reports them, each with the name a step takes when it is given none.  bench.py and
// tools/bench_*.py match on the numbers, so a kind keeps its number.
#define B2_STEP_KINDS(X)                                                                                              \
  X(kStepConv, 0, "conv") X(kStepStemPack, 1, "stem_pack") X(kStepMaxpool, 2, "maxpool")                          \
  X(kStepP6Subsample, 3, "p6_subsample") X(kStepRpnProposals, 4, "rpn_proposals")                                 \
  X(kStepRoialignProposals, 5, "roialign_proposals") X(kStepHeadPost, 6, "head_post")                            \
  X(kStepRoialignFinal, 7, "roialign_final") X(kStepRoialignMask, 8, "roialign_mask")                            \
  X(kStepMaskSelect, 9, "mask_select") X(kStepGnStats, 10, "gn_stats") X(kStepGnApply, 11, "gn_apply")            \
  X(kStepGnRoi, 12, "gn_roi") X(kStepSeSqueeze, 13, "se_squeeze") X(kStepSeExcite, 14, "se_excite")               \
  X(kStepSeApply, 15, "se_apply") X(kStepRelationAttend, 16, "relation_attend") X(kStepDeformSample, 17, "deform_sample") \
  X(kStepAttPool, 18, "att_pool") X(kStepAttSum, 19, "att_sum") X(kStepSoSelect, 20, "so_select")             \
  X(kStepSoGather, 21, "so_gather") X(kStepSoRoialign, 22, "so_roialign") X(kStepSoAttend, 23, "so_attend")       \
  X(kStepSoFinish, 24, "so_finish")
enum StepKind {
#define B2_STEP_KIND_VALUE(e, v, n) e = v,
  B2_STEP_KINDS(B2_STEP_KIND_VALUE)
#undef B2_STEP_KIND_VALUE
};

// Everything the builders read and append to.
struct DetPlan {
  Arena arena;             // first member: freed after everything that refers to it
  bool split = false;      // (hi, lo) planes, else fp16 only
  int conv_impl = 0;       // 0 tensor cores, 1 CUDA cores
  int acc_kb = 0;          // ConvDesc::acc_kb of every conv
  int batch = 1;           // images of a full-batch launch
  // the forked phases 0-2 run as nsplit batch parts on as many streams (dual = nsplit > 1): their steps get one launch
  // per part
  bool dual = false;
  int nsplit = 1;
  unsigned int* range_flag = nullptr;          // ORed by convs and GroupNorm outputs beyond the fp16 range; nullptr = off
  std::vector<std::unique_ptr<ConvLayer>> layers;
  std::vector<ConvLayer*> part_layers;         // layers of the forked phases 0-2 (they get per-part plans)
  std::vector<std::unique_ptr<GnOp>> gns;
  std::vector<std::unique_ptr<SeOp>> ses;
  std::vector<std::unique_ptr<RelOp>> rels;
  int att_channels = 0;    // ROI channels of the attention box head (add_att_head); 0 = none
  std::vector<Step> steps;
  StageMap stages;
  // the scratch all relation modules share: query|key [Mpad][2D] fp32, P [B][16K][Kp], P.V = the output_linear operand
  // [Mpad][16D]
  float* rel_qk = nullptr;
  Planes rel_p, rel_o;

  bool alloc_planes(Planes& p, int B, int H, int W, int C) {
    p = arena.planes(B, H, W, C, split);
    return p.hi != nullptr;
  }
  // M rows of C channels: a [1][1][M][C] view of planes padded to whole 128-row tiles (the box head's row buffers)
  bool alloc_rows(Planes& p, int M, int C) {
    if (!alloc_planes(p, 1, 1, (M + 127) / 128 * 128, C)) return false;
    p.W = M;
    return true;
  }
};

// Adds step `kind` of `phase`.  `launch(b0, n, st)` enqueues it over images [b0, b0 + n); in the forked phases 0-2 the
// step gets one launch per batch part.  An empty name is the kind's name.
Step& add_batch_step(DetPlan& p, int phase, StepKind kind, const std::string& name,
                     const std::function<int(int, int, cudaStream_t)>& launch, int launches = 1);

// A conv of R x R taps to Cout channels; the caller sets the other fields of the geometry and epilogue.
inline ConvDesc conv_desc(int R, int Cout) {
  ConvDesc d;
  d.R = d.S = R;
  d.Cout = Cout;
  return d;
}
// The same zero padding on all four sides.
inline void pad_all(ConvDesc& d, int pad) { d.pad_t = d.pad_b = d.pad_l = d.pad_r = pad; }
// TF padding SAME of a 3x3 conv at d.stride / d.dil over an h x w input.
void same_pads3(int h, int w, ConvDesc& d);

// Adds the conv `name` reading `in` (the d.in_H x d.in_W view, 0 = the whole buffer; pixel stride d.in_ld, 0 = in.C) and
// writing the planes `out`, with `res` (read at (y >> d.res_shift, x >> d.res_shift)) added in the epilogue when given.
ConvLayer* add_conv(DetPlan& p, int phase, const std::string& name, const Planes& in, ConvDesc d, ConvAffine affine,
                    const Planes& out, const Planes* res = nullptr, Layout layout = kHwio);
// A dense layer that runs `src`'s packed weights and epilogue (bias, ReLU) over other rows: `in` has src's input width
// (nullptr with the error set otherwise).
ConvLayer* add_conv_shared(DetPlan& p, int phase, const std::string& name, const Planes& in, const ConvLayer& src,
                           const Planes& out);
// The same with an fp32 output: rows of stride `ldc` at `out_f32`.
ConvLayer* add_conv_f32(DetPlan& p, int phase, const std::string& name, const Planes& in, ConvDesc d, ConvAffine affine,
                        float* out_f32, int ldc, Layout layout = kHwio);

// GroupNorm `name` of the view (view_h x view_w at (off_h, off_w)) of `buf`, in place, then + `res` (read at
// (y >> res_shift, x >> res_shift)) and ReLU; with per_roi one step that normalises each [7][7][C] sample on chip.
int add_gn(DetPlan& p, int phase, const std::string& name, const Planes& buf, int view_h, int view_w, int off_h, int off_w,
           const Planes* res, int res_shift, bool relu, bool per_roi = false);
// Squeeze-excite of the bottleneck `name` on its conv3 output `buf`, then relu(buf * gate + res) in place (`res` may be
// null).  The gate lands in the SeOp it records.
int add_se(DetPlan& p, int phase, const std::string& name, const Planes& buf, const Planes* res);
// The relation module `name` over the B*K head rows h (image b's rows at b*K, D columns) with the proposals `boxes`
// [B][K][4] and `count` [B] on the device: out = h + output_linear(P . h).
int add_relation(DetPlan& p, const std::string& name, int B, int K, int D, const float* boxes, const int* count,
                 const Planes& h, const Planes& out);
// person_object_relation `scope` (nn.py:194-270, use_so_association) over `rows` ([C * Rq + Tp][D] planes: C blocks of Rq
// query rows, then Tp key rows) with their boxes [C * Rq + Tp][4] on the device; *kq query rows of each block and *nref
// key rows are valid (device ints).  out ([C * Rq][D]) = query rows + output_linear(P . key rows).
int add_so_association(DetPlan& p, int phase, const std::string& scope, int C, int Rq, int Tp, const float* boxes,
                       const int* kq, const int* nref, const Planes& rows, const Planes& out);
// The attention branch of the class-specific box head (use_att_frcnn_head) over the head rows `hidden` ([M][D] rows):
// out = hidden + relu(att_trans(sum over the 49 bins of roi)), roi the ROIAlign planes [M][49][C]; `pooled` ([M][C]) and
// `att` ([M][D]) are its intermediate rows.
int add_att_head(DetPlan& p, const Planes& roi, int C, const Planes& hidden, const Planes& pooled, const Planes& att,
                 const Planes& out);
// The deformable conv2 of block `name` from conv1's output `in` into `out` ([B][ceil(H/2)][ceil(W/2)][in.C]).
int add_deform(DetPlan& p, const std::string& name, const Planes& in, const Planes& out);

// The planes the mask head writes, [M][14][14][C] each (M = B * R boxes, C = 256) but up ([M][14][14][4C], the deconv's
// (tap, channel) outputs).  The layers may share buffers as long as none reads the one it writes: the engine ping-pongs
// two (roi = fcn[1] = fcn[3], fcn[0] = fcn[2]).
struct MaskBufs {
  Planes roi, fcn[4], up;
};
// The class conv's output of M boxes: 784 rows per box (196 pixels x 4 taps), padded to whole 128-row tiles, of
// mask_logits_ld(num_class) fp32 columns.
inline size_t mask_logits_rows(int M) { return (static_cast<size_t>(M) * 784 + 127) / 128 * 128; }
inline int mask_logits_ld(int num_class) { return (num_class - 1 + 15) / 16 * 16; }
// The mask head (models.py:934-961, 1173-1199), phase 7, over the B x R boxes of `roi` (its levels, boxes and count;
// the outputs are set here): ROIAlign 14 into buf.roi, maskrcnn/fcn0..3 (3x3 SAME + bias + ReLU) into buf.fcn, the
// transposed conv maskrcnn/deconv into buf.up, the class conv maskrcnn/conv into `logits` and the sigmoid of each box's
// own class (labels [B][R], 1 .. num_class - 1 below the count) into masks [B][R][28][28].
int add_mask_head(DetPlan& p, RoiAlignParams roi, int num_class, const MaskBufs& buf, const int* labels, float* logits,
                  float* masks);

// The planes a residual block writes: conv1's output, conv2's (bottleneck only), the projection shortcut's (used when
// the input's width is not the block's) and the block output.
struct BlockBufs {
  Planes t1, t2, sc, out;
};
// The basic block `name` (ResNet-18 / 34) from `x` at `stride`; GroupNorm steps with gn, else BatchNorm epilogues.
int add_basic_block(DetPlan& p, const std::string& name, const Planes& x, int stride, const BlockBufs& buf, bool gn);
// The bottleneck `name` from `x` at `stride` and conv2 dilation `dil`: GroupNorm steps with gn, else BatchNorm epilogues;
// squeeze-excite before the residual sum with se, the grouped 32x4d conv2 with rx, the deformable conv2 with deform.
int add_bottleneck(DetPlan& p, const std::string& name, const Planes& x, int stride, int dil, const BlockBufs& buf, bool gn,
                   bool se, bool rx, bool deform);

// The full-batch tensor-core plan of every layer and, with dual, each forked layer's per-part plans (conv_impl 0 only).
int plan_layers(DetPlan& p, int num_sms);
// Every layer, GroupNorm, squeeze-excite and relation module of the plan from the checkpoint `ws`, and the attention head's
// weight check; num_class is the
// checkpoint's class count of the fused box-head outputs.  With num_partial > 0 those outputs keep the class-0 column and
// the columns of partial_ids[0 .. num_partial), in that order (use_partial_classes).
int load_weights(const DetPlan& p, const WeightSet& ws, int num_class, cudaStream_t st, const int* partial_ids = nullptr,
                 int num_partial = 0);

}  // namespace b2
