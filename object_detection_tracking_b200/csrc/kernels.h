// Parameter blocks and launchers of the non-GEMM kernels (proposals, ROIAlign, detection post-process,
// appearance cost).  All launches are asynchronous on the given stream; nothing syncs with the host.
#pragma once
#include <vector>

#include "common.h"

struct b2_masks;

namespace b2 {

// stem.cu
int f32_to_planes(const float* src, __half* hi, __half* lo, size_t n, cudaStream_t s);
int planes_to_f32(const __half* hi, const __half* lo, float* dst, size_t n, cudaStream_t s);
int resize_u8_launch(const uint8_t* src, int B, int sh, int sw, float* dst, int dh, int dw, cudaStream_t s);
// operand of the ReID stems: [B][Hu][Wu][64] from RGB uint8 crops, torchvision ToTensor + Normalize (x / 255 - mean) / std
// with RGB constants (feature_extractor.py:190-196), pad 3 on every side (stem.cu)
int stem_pack_launch(const uint8_t* img, int B, int H, int W, __half* out_hi, __half* out_lo, int Hu, int Wu,
                     cudaStream_t s);
// compact operand of the detector stem: [B][Hu][Wv = Wu + 3][16] from uint8 (is_u8) or float32 BGR frames,
// (x * (1/255) - mean) / std with BGR constants (models.py:345-355), pad [3, 2 + pad-to-32] (stem.cu)
int stem_pack16_launch(const void* img, int is_u8, int B, int H, int W, __half* out_hi, __half* out_lo, int Hu, int Wv,
                       cudaStream_t s);
// reid_ingest.cu: track boxes [n][5] (frame, x, y, w, h; int32, device) of uint8 BGR frames [nf][H][W][3] -> RGB uint8
// crops [n][out_h][out_w][3] resized as Pillow's Image.resize(BILINEAR) (pil_resize_math.h); out_w <= 256.  The boxes must
// have passed reid_boxes_check (host copy of the same table): frame index in [0, nf), w, h >= 1, inside the frame.
int reid_boxes_check(const int32_t* boxes_host, int n, int nf, int H, int W, const char* who);
int reid_crop_resize_launch(const uint8_t* frames, int H, int W, const int32_t* boxes, int n, uint8_t* crops, int out_h,
                            int out_w, cudaStream_t s);
// mask_rle.cu: a grow-only device buffer (reserve() synchronises `s` before it replaces a smaller one), the workspaces of
// a b2_masks encoder
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf();
  int reserve(size_t bytes, cudaStream_t s);
};
// Return code of the mask calls for a refused input (bad box, size or shape), checked on the host before any launch.
constexpr int kMaskRefused = -2;
// The RLE of b2_masks_encode on stream s: masks [n][28][28] float32 (device memory of the encoder's GPU when
// masks_on_device, else host), boxes [n][4] host.  Fills offsets[n + 1], copies the strings into bytes when capacity
// holds them and keeps them in the encoder for b2_masks_fetch.
int mask_encode(b2_masks* e, const float* boxes, const float* masks, int masks_on_device, int n, int mask_h, int mask_w,
                int H, int W, int64_t* offsets, char* bytes, int64_t capacity, cudaStream_t s, const char* who);
int mask_encoder_device(const b2_masks* e);
// 3x3 stride-2 max-pool, window rows 2y - 1 .. 2y + 1 (columns alike) clipped to the map, Ho x Wo chosen by the caller;
// C a multiple of 8.  The running maximum starts from 0, so this is the max-pool only of inputs >= 0: every caller feeds
// it post-ReLU data.  The output is the (hi, lo) pair of the element with the largest joined value.
int maxpool_launch(const __half* in_hi, const __half* in_lo, int B, int H, int W, int C, __half* out_hi,
                   __half* out_lo, int Ho, int Wo, cudaStream_t s);

// rpn.cu
struct RpnParams {
  const float* logits[5];   // per level [B * h*w][16]: cols 0..2 objectness, 3..14 deltas (anchor-major)
  int h[5], w[5];
  float stride[5];
  float cell[5][3][4];      // cell anchors x1,y1,x2,y2 (generate_anchors.py semantics, before the +1)
  int B, topk;
  float img_h, img_w, decode_clip, min_size, nms_thr;
  int multi;                // batch-graph semantics: no min-size filter, zero-padded merge, zero-area drop
  float* lvl_boxes;         // [B][5][topk][4]
  float* lvl_scores;        // [B][5][topk]
  int* lvl_count;           // [B][5]
  float* prop_boxes;        // [B][topk][4]
  float* prop_scores;       // [B][topk]
  int* prop_count;          // [B]
};
int rpn_proposals_launch(const RpnParams& p, cudaStream_t s);

// roialign.cu
struct RoiAlignParams {
  const __half* feat_hi[4];   // p2..p5, NHWC
  const __half* feat_lo[4];   // nullptr in fp16 precision
  int H[4], W[4];             // cropped view the ROIAlign sees (models.py:382-390)
  int pitch_H[4], pitch_W[4]; // buffer dims
  float inv_stride[4];
  int C;                      // 256
  int B, rois_per_image;      // boxes [B][rois_per_image][4], count[B]
  const float* boxes;
  const int* count;
  __half* out_hi;             // [B*rois][7][7][C]   (fc6 operand order), or
  __half* out_lo;
  float* out_nchw;            // [B*rois][C][7][7]   fp32 (fpn_box_feat contract)
  int out_res;                // 0 / 7: 7x7 bins from a 14x14 crop; 14: 14x14 bins from a 28x28 crop (mask head,
                              // models.py:936-937), planes output [B*rois][14][14][C]
  int one_image;              // 1: the B box groups are groups of one image, all read the features of image 0
};
int roialign_launch(const RoiAlignParams& p, cudaStream_t s);

// mask_head.cu: the mask head's output (models.py:950-958).  out [B*R][28][28] = sigmoid of channel labels[roi] - 1 of
// the class-conv logits ([B*R*196*4][ld] fp32, rows (roi * 196 + (Y >> 1) * 14 + (X >> 1)) * 4 + (Y & 1) * 2 + (X & 1)),
// 0 for rows j >= count[b].  The labels below the count must lie in 1 .. Cout of the class conv: the device does not check
// them.
int mask_select_launch(const float* logits, int ld, const int* labels, const int* count, int B, int R, float* out,
                       cudaStream_t s);

// head.cu
struct HeadPostParams {
  const float* logits;        // [B*rois][ld]: cols 0..nc-1 class logits, nc + c*4 .. box logits of class c
  int ld, num_class, B, rois_per_image;
  int class_agnostic;         // box logits shared by all classes (use_frcnn_class_agnostic)
  const float* rois;          // [B][rois][4]
  const int* roi_count;       // [B]
  float reg_w[4];
  float decode_clip, img_h, img_w, score_thresh, nms_thr;
  int max_per_class, max_total;
  float* probs;               // [B][rois][num_class]
  float* dec_boxes;           // [B][rois][num_class-1][4]
  int* cls_keep;              // [B][num_class-1][max_per_class] roi indices
  int* cls_count;             // [B][num_class-1]
  float* final_boxes;         // [B][max_total][4]
  float* final_probs;         // [B][max_total]
  int* final_labels;          // [B][max_total]
  int* final_count;           // [B]
  // use_bg_score (models.py:1263-1270): null = no filter.  Else [B][rois]: row i's rank j among the image's rows below
  // roi_count[b] whose argmax over probs is not column 0, or -1 for a dropped row.  The per-class NMS skips the dropped
  // rows, and the final top-k gathers dec_boxes at row j instead of i, as the reference's gather_nd on the unfiltered
  // boxes does (models.py:925-930)
  int* bg_rank;
};
int head_post_launch(const HeadPostParams& p, cudaStream_t s);
// head_post_launch's selection alone, over p.probs and p.dec_boxes as they stand: with p.bg_rank the background filter,
// then per-class NMS, then the final top-k
int head_select_launch(const HeadPostParams& p, cudaStream_t s);
// the per-class NMS of classes c0 .. c0 + n - 1 (dec_boxes column c, probs column c + 1) alone
int class_nms_launch(const HeadPostParams& p, int c0, int n, cudaStream_t s);

// small_objects.cu -- the small-object branch of the single-image graph (use_small_object_head, models.py:590-692,
// 845-897).  Rows of the branch: C blocks of R rows (small class i's boxes in NMS selection order) then Tp person rows.
struct SoParams {
  // so_select: the head's outputs for the B = 1 image
  const float* logits;        // [rois][ld] head logits (HeadPostParams layout)
  int ld, num_class, rois;
  const float* roi_boxes;     // [rois][4] proposals
  const int* roi_count;       // [1]
  const float* probs;         // [rois][num_class] the head's softmax
  float reg_w[4];
  float decode_clip, img_w, img_h;
  int C, R, Tp;               // small classes, rows per class block (result_per_im), person rows (0 = no association)
  int ids[81];                // the head class ids of the C small classes, then Person's when Tp > 0
  float* sel_probs;           // [rois][C + 2]: column s + 1 the probability of selected class s (Person last)
  float* sel_boxes;           // [rois][C + 1][4] unclipped decoded boxes of the selected classes
  // so_gather: the selections (HeadPostParams cls_keep / cls_count of the two NMS launches)
  const int* keep;            // [C][R] small classes
  const int* person_keep;     // [Tp] Person
  const int* sel_count;       // [C + 1] kept per class, Person last
  float* rows_boxes;          // [C * R + Tp][4] the branch's rows, unclipped, zero beyond the counts
  int* row_count;             // [C + 1]: K for every small class block, then the person rows
  int* k;                     // [1] K: the common count, 0 when the classes kept different counts
  int* status;                // [1] 0, or 1 when the counts differed
  // so_finish: the classification layer's fp32 output [C * R][ldl], row block i's columns 2i, 2i + 1
  const float* cls_logits;
  int ldl;
  float* fin_logits;          // [R][C + 1] the rebuilt logits (models.py:675-681)
  float* fin_boxes;           // [R][C][4] the rows' boxes clipped to the image
};
int so_select_launch(const SoParams& p, cudaStream_t s);
int so_gather_launch(const SoParams& p, cudaStream_t s);
int so_finish_launch(const SoParams& p, cudaStream_t s);

// person_object_relation (nn.py:194-270) over C blocks of Rq query rows and Tp key (person) rows: P [C * Rq * 16][Tpp]
// planes (row q * 16 + g) of softmax_j(log(max(wg, 1e-6)) + q_g . k_g / sqrt(D / 16)) over the first *nref key rows, and
// the key rows' V^T [D][Tpp] (the P.V layer's weights).  Query rows at or beyond *kq of their block, and all rows when
// *nref is 0, are zero.
struct SoAttendParams {
  const float* boxes;         // [C * Rq + Tp][4]: query boxes, then key boxes
  const int* kq;              // [1] valid query rows per block
  const int* nref;            // [1] valid key rows
  const float* qk;            // [C * Rq + Tp][ldqk] fp32: query in columns [0, D), key in [D, 2D)
  int ldqk, D, C, Rq, Tp, Tpp, rows;
  const float* geo;           // kRelGeoWeights (relation_upload_geo)
  const __half* v_hi;         // the key rows' features [Tp][D] planes: the value
  const __half* v_lo;
  __half* p_hi;
  __half* p_lo;
  __half* vt_hi;              // [D][Tpp]
  __half* vt_lo;
};
int so_attend_launch(const SoAttendParams& p, cudaStream_t s);

// groupnorm.cu -- GroupNorm of a conv output at run time (nn.py:81-108), 32 groups, eps 1e-5
struct GnParams {
  const __half* x_hi;         // input planes (NHWC); the view is H x W at (off_h, off_w) of a pitch_H x pitch_W buffer
  const __half* x_lo;         // nullptr in fp16 precision
  __half* y_hi;               // output planes, same geometry as x (may be x: in place); only the view is written
  __half* y_lo;
  int B, H, W, C;             // images (ROIs for gn_roi), view extents, channels
  int pitch_H, pitch_W, ld, off_h, off_w;
  const __half* r_hi;         // optional residual added after the normalisation: pixel (y >> res_shift, x >> res_shift)
  const __half* r_lo;         // of a res_H x res_W buffer with pixel stride res_ld (res_shift 1 = nearest 2x upsample)
  int res_H, res_W, res_ld, res_shift;
  int relu;                   // ReLU after the (normalise, residual) sum
  const float* gamma;         // [C]
  const float* beta;          // [C]
  const float* gate;          // se_apply only: [B][C] per-image channel gate, y = x * gate[b][c] (+ residual) (ReLU)
  int chunks;                 // pixel chunks per image (gn_chunks): blocks per image of gn_stats / gn_apply / se_apply
  float* partial;             // [B][chunks][32][3] (count, mean, M2) per chunk and group
  float* stats;               // [B][32][2] (mean, var) per image and group
  unsigned int* counter;      // [B] finished-chunk tickets, zero between launches
  unsigned int* range_flag;   // ORed with 1 when an output leaves the fp16 range (nullptr = not monitored)
};
int gn_chunks(int H, int W, int C);
int gn_stats_launch(const GnParams& p, cudaStream_t s);
int gn_apply_launch(const GnParams& p, cudaStream_t s);
int gn_roi_launch(const GnParams& p, cudaStream_t s);   // per sample statistics + apply in one kernel (7x7 ROI maps)
// The squeeze-excite gate of the SE-ResNet bottleneck through GroupNorm's apply path (scale = p.gate[b], shift 0);
// p.gamma / p.beta unused
int se_apply_launch(const GnParams& p, cudaStream_t s);

// reid.cu
int dwconv3x3_launch(const __half* in_hi, const __half* in_lo, int B, int H, int W, int C, const float* w,
                     const float* bias, __half* out_hi, __half* out_lo, cudaStream_t s);
int gap_launch(const __half* in_hi, const __half* in_lo, int B, int HW, int C, float* out, int out_ld, cudaStream_t s);
int gate_mlp_launch(const float* g, int rows, int C, int Creal, int Cr, const float* w1, const float* b1,
                    const float* w2, const float* b2, float* gates, cudaStream_t s);
int gated_sum4_launch(const __half* const hi[4], const __half* const lo[4], const float* gates, int B, int HW, int C,
                      __half* out_hi, __half* out_lo, cudaStream_t s);
int avgpool2_launch(const __half* in_hi, const __half* in_lo, int B, int H, int W, int C, __half* out_hi,
                    __half* out_lo, cudaStream_t s);

// effdet.cu -- EfficientDet feature network, heads' depthwise halves, post-processing
struct BifpnInput {
  const __half* hi;
  const __half* lo;
  int H, W;               // source map size
  int mode;               // 0 same size, 1 max-pool 3x3/2 SAME from a 2x finer map, 2 nearest 2x upsampling
  int pad_t, pad_l;       // SAME padding of mode 1
  float weight;           // fast-attention edge weight relu(w_i)
};
struct BifpnCombineParams {
  BifpnInput in[3];
  int n_in;
  int B, Ho, Wo, C;
  int weighted;           // 1: node = sum_i x_i * w_i / denom (fastattn); 0: plain sum
  float denom;            // sum_i relu(w_i) + 1e-4
  int swish;              // apply x * sigmoid(x) to the combined node (op_after_combine input)
  __half* out_hi;
  __half* out_lo;
};
// Input i of a node of size th x tw from a source map H x W: the resampling mode from the two sizes, and mode 1's pads
int bifpn_set_input(BifpnInput& bi, const __half* hi, const __half* lo, int H, int W, int th, int tw);
// fastattn: weight_i = relu(raw_i), denom = add_n(weights) + 1e-4, in float32 as build_bifpn_layer computes them
void bifpn_set_weights(BifpnCombineParams& p, const float* raw);
int bifpn_combine_launch(const BifpnCombineParams& p, cudaStream_t s);
int dw3x3_plain_launch(const __half* in_hi, const __half* in_lo, int B, int H, int W, int C, const float* w, __half* out_hi,
                       __half* out_lo, cudaStream_t s);

// Every buffer below holds one slice per image (B images; the image is a grid dimension of every kernel): head outputs
// image b at logits[l] + b * logit_bstride[l] (boxes alike), the scratch and the outputs at b times their per-image size.
struct EffdetPostParams {
  const float* logits[5];   // per level [B][h*w][ld]: anchor-major, class-minor (A * num_classes real columns)
  const float* boxes[5];    // per level [B][h*w][ldb]: A * 4 (ty, tx, th, tw)
  unsigned long long logit_bstride[5], box_bstride[5];   // elements between consecutive images of logits[l] / boxes[l]
  int B;
  int ld[5], ldb[5], w[5];
  unsigned long long level_off[6];   // flat logit index where each level starts
  unsigned long long total;
  int n_levels, anchors, num_classes, min_level;
  double stride_y[5], stride_x[5], half_y[5][9], half_x[5][9];   // anchor grid (anchors.py:216-257), float64 like numpy
  int k, max_out;
  float score_thresh, nms_thr;
  unsigned int* hist;       // [B][256]
  uint32_t* state;          // [B][8]: prefix, mask, need, n_selected (> k-th), n_ties (== k-th), n_candidates
  unsigned long long* cand; // [B][k]
  unsigned long long* ties; // [B][k] lowest-index ties of the k-th value
  unsigned int* tie_cnt;    // [B][effdet_topk_blocks()] ties per block (blocks own contiguous index ranges)
  unsigned int* tie_off;    // exclusive prefix of tie_cnt
  float4* cand_box;         // [B][k] (ymin, xmin, ymax, xmax), score order
  float* cand_score;
  int* cand_cls;
  int* cand_lvl;
  unsigned long long* mask; // [B][k][ceil(k/64)]
  float4* out_boxes;        // [B][max_out] x1 y1 x2 y2, scaled back to the original frame
  float* out_scores;
  int* out_classes;
  int* out_levels;
  int* out_count;           // [B]
};
int effdet_topk_blocks();
// image_scale_dev [B]: image b's boxes are multiplied by image_scale_dev[b]
int effdet_post_launch(const EffdetPostParams& p, const float* image_scale_dev, cudaStream_t s);

// effnet.cu -- EfficientNet backbone pieces + EfficientDet input pre-processing
// One image of a pre-processing launch: its BGR frame at byte `src` of the upload buffer, h x w, resized to sh x sw
// (ys = h / sh, xs = w / sw in float32, as effnet_frame computes them)
struct EffnetFrame {
  unsigned long long src;
  int h, w, sh, sw;
  float ys, xs;
};
EffnetFrame effnet_frame(unsigned long long src, int h, int w, int sh, int sw);
// frames (device table of B entries) -> out [B][H][W][3] fp32
int effnet_preprocess_launch(const uint8_t* frames, const EffnetFrame* table, int B, float* out, int H, int W, cudaStream_t s);
int stem_im2col_launch(const float* img, int B, int H, int W, int Ho, int Wo, int pad_t, int pad_l, __half* out_hi,
                       __half* out_lo, cudaStream_t s);
struct DwConvParams {
  const __half* in_hi;
  const __half* in_lo;
  int B, H, W, C;           // input map [B][H][W][C], C multiple of 8
  int K, stride, pad_t, pad_l;
  int Ho, Wo;
  const float* w;           // [K*K][C], BatchNorm scale folded in
  const float* bias;        // [C], BatchNorm shift
  __half* out_hi;
  __half* out_lo;
};
int dwconv_bn_swish_launch(const DwConvParams& p, cudaStream_t s);
int dwconv_launch(const DwConvParams& p, int act, cudaStream_t s);   // act 0 none / 2 swish; p.bias may be null
int se_chunks(int HW);      // rows of the partial-sum buffer se_gate_launch needs
int se_fc1_parts();         // rows of the r_part buffer (row stride se_max_nr())
int se_max_nr();
// MBConv's squeeze-excite over B images, each gate folded into its own copy of the projection weights: w [rows][Cpad]
// fp32 -> (w_hi, w_lo) [B][rows][Cpad]
int se_gate_launch(const __half* in_hi, const __half* in_lo, int B, int HW, int Cpad, int C, int nr, float* partial,
                   float* r_part, const float* w1, const float* b1, const float* w2, const float* b2, float* gate,
                   const float* w, int rows, __half* w_hi, __half* w_lo, cudaStream_t s);
// The two halves of squeeze-excite over B images [B][HW][Cpad], every image with its own scratch: partial
// [B][se_chunks(HW)][Cpad], r_part [B][se_fc1_parts()][se_max_nr()], gate [B][Cpad].  relu selects the hidden activation
// (1 ReLU for the SE-ResNet bottleneck, 0 swish for MBConv); w == nullptr writes the gate only (no weight fold), else
// image b's folded weights go to w_hi / w_lo + b * rows * Cpad.
int se_squeeze_launch(const __half* in_hi, const __half* in_lo, int B, int HW, int Cpad, float* partial, cudaStream_t s);
int se_excite_launch(const float* partial, int B, int HW, int Cpad, int C, int nr, float* r_part, const float* w1,
                     const float* b1, const float* w2, const float* b2, int relu, float* gate, const float* w, int rows,
                     __half* w_hi, __half* w_lo, cudaStream_t s);

// roialign.cu -- ROIAlign 7x7 on the detection's own level + mean over the 49 bins (efficientdet_wrapper.py:265-301)
struct LevelRoiFeatParams {
  const __half* feat_hi[5]; // per level [B][H][W][C]
  const __half* feat_lo[5];
  int H[5], W[5];
  float inv_stride[5];
  int B, C, Creal, min_level, max_out;
  const float4* boxes;      // [B][max_out] x1 y1 x2 y2
  const int* levels;        // [B][max_out]
  const int* count;         // [B]
  float* out;               // [B][max_out][Creal]
};
int level_roi_feat_launch(const LevelRoiFeatParams& p, cudaStream_t s);

// relation.cu -- the box head's relation module (add_relation_nn, nn.py:115-190): the geometry + attention softmax and
// the V^T operand of the per-image P.V layer; query / key, P.V and output_linear run on conv_tc_kernel
constexpr int kRelGroups = 16, kRelGeoDim = 64;
constexpr int kRelGeoWeights = 4 * kRelGeoDim + kRelGeoDim + kRelGeoDim * kRelGroups + kRelGroups;
struct RelationParams {
  const float* boxes;       // [B][K][4] proposals x1 y1 x2 y2
  const int* count;         // [B] proposals per image (rows j >= count are padding)
  const float* qk;          // [B*K][ldqk] fp32: query in columns [0, D), key in [D, 2D)
  int ldqk, D, K, Kp;       // Kp: K rounded up to 64 (columns of P, rows of V^T)
  int rows;                 // query rows per block (relation_rows_per_block)
  const float* geo;         // kRelGeoWeights: geo_emb W [4][64], b [64], geo_conv W [64][16], b [16]
  const __half* h_hi;       // h [B*K][D] planes: the value
  const __half* h_lo;
  __half* p_hi;             // P [B][K*16][Kp] planes, row i * 16 + g
  __half* p_lo;
  __half* const* vt_hi;     // device table of B pointers: image b's V^T [D][Kp] planes (the P.V layer's weights)
  __half* const* vt_lo;
};
int relation_rows_per_block(int Kp, int D);
// V^T and P of images [b0, b0 + n)
int relation_attend_launch(const RelationParams& p, int b0, int n, cudaStream_t s);
// query_linear / key_linear W [D][D] ([in, out]) -> the fused layer's [2D][D] operand
void relation_pack_qk(const float* wq, const float* wk, int D, std::vector<float>& packed);
// geo_emb W [4, 64], b [64], geo_conv W [1, 1, 64, 16], b [16] -> dst (kRelGeoWeights floats on the device)
int relation_upload_geo(const float* emb_w, const float* emb_b, const float* conv_w, const float* conv_b, float* dst,
                        cudaStream_t s);

// att_head.cu -- the attention box head's pool (use_att_frcnn_head, models.py:1064-1089): ROIAlign rows [M][49][C] planes
// -> [M][C] planes, the sum over the 49 bins in bin order; a ROI with a non-finite input gets an all-NaN row.  A finite
// sum beyond +-65504 ORs *range_flag (nullptr = not monitored)
int att_pool_launch(const __half* in_hi, const __half* in_lo, int M, int C, __half* out_hi, __half* out_lo,
                    unsigned int* range_flag, cudaStream_t s);

// deform.cu -- the bilinear sampler of a deformable conv2 (use_deformable, deformable_helper.py:42-137): conv1's output
// sampled at tap k's base + offset around (2i, 2j), clamped to the map, into the operand of a 1x1 conv with K = 9 * C
constexpr int kDeformOffsetLd = 32;   // row stride of the fp32 offsets: the offset conv's 18 outputs padded to Cout_pad
struct DeformParams {
  const __half* in_hi;      // conv1 output [B][H][W][C] planes
  const __half* in_lo;
  const float* offset;      // [B][Ho][Wo][ld_off] fp32: column 2k the y, 2k + 1 the x offset of tap k
  int ld_off;
  int H, W, C, Ho, Wo;      // Ho = ceil(H / 2), Wo = ceil(W / 2); C a multiple of 8
  __half* out_hi;           // [B][Ho][Wo][9][C] planes: tap-major, then channel
  __half* out_lo;
};
// images [b0, b0 + n)
int deform_sample_launch(const DeformParams& p, int b0, int n, cudaStream_t s);

// cosine.cu
int cosine_normalize_rows(const float* src, int rows, int D, float eps, __half* hi, __half* lo, int ld, cudaStream_t s);
int rows_to_planes(const float* src, int rows, int D, __half* hi, __half* lo, int ld, float* sqnorm,
                   unsigned int* range_flag, cudaStream_t s);
int distance_finish(const float* dots, int ld, int na, int nb, int metric, const float* na2, const float* nb2, float* out,
                    cudaStream_t s);
int pair_segmin(const float* dots, int ld, const float* na2, const float* nb2, const int* seg_a, int N, const int* seg_b,
                int M, const unsigned char* gate, float fill, float* out, cudaStream_t s);
int cosine_segmin(const float* dots, int ld, const int* seg_offsets, int T, int N, float* cost, cudaStream_t s);
// out[p] = min over the block (query segment pairs[2p], gallery segment pairs[2p+1]) of (na2 + nb2) - 2 dots, unclamped
int tracklet_pair_min(const float* dots, int ld, const float* na2, const float* nb2, const int* seg_q, const int* seg_g,
                      const int* pairs, int P, float* out, cudaStream_t s);
// mean [S][D] of the rows of src [seg[S]][D] per segment: float32 sum in row order / count
int segment_mean(const float* src, const int* seg, int S, int D, float* mean, cudaStream_t s);

}  // namespace b2
