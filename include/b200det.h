/* libb200det -- C ABI of the H100-native detect -> embed -> associate hot path.
 *
 * Drop-in boundary for JunweiLiang/Object_Detection_Tracking: the entry points below are what the
 * reference's Python call surface binds for this path (the reference has no native code of its own;
 * its hot path is `sess.run` on a TF graph).  Citations are file:line in the reference repository.
 *
 *   models.get_model(config, gpuid, ...)                       models.py:97-119      -> b2_create + b2_load_weights
 *   model.get_feed_dict_forward(img) + sess.run([final_boxes,
 *       final_labels, final_probs, fpn_box_feat], feed_dict)   obj_detect_tracking.py:610-635,
 *                                                              models.py:1629-1636   -> b2_detect_host / b2_detect
 *   model.get_feed_dict_forward_multi(imgs) + sess.run         models.py:3301-3310,
 *                                                              obj_detect_tracking_multi_queuer.py:474-480 -> same, batch > 1
 *   initialize(load=True, ...) (.npz / ckpt name->array load)  obj_detect_tracking.py:392-448 -> b2_load_weights
 *   NearestNeighborDistanceMetric.distance(features, targets)  deep_sort/nn_matching.py:156-177 -> b2_cosine_cost
 *
 * Conventions: every function returns 0 on success, <0 on error (message via b2_last_error()); no
 * exceptions cross the ABI; plain pointers and sizes only.  A b2_ctx is bound to one device and is
 * single-threaded (the reference calls sess.run from exactly one thread).  The library never
 * allocates caller-visible output memory: callers pass capacity-sized buffers and receive counts.
 */
#ifndef B200DET_H_
#define B200DET_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b2_ctx b2_ctx;

/* Mirrors the fields of the reference's argparse namespace that shape the inference graph
 * (obj_detect_tracking.py:236-389). */
typedef struct b2_config {
  int32_t batch;              /* im_batch_size; frames per b2_detect call */
  int32_t height, width;      /* frame size after resizeImage (nn.py:1540-1560), e.g. 720 x 1280 */
  int32_t input_dtype;        /* 0 = float32 HWC BGR (the reference placeholder), 1 = uint8 HWC BGR */
  int32_t num_class;          /* incl. background (15 ActEV, 81 COCO) */
  int32_t resnet_blocks[4];   /* (3,4,23,3) R101, (3,4,6,3) R50 */
  int32_t use_dilations;      /* --version 3: res5 dilation 2 */
  int32_t class_agnostic;     /* use_frcnn_class_agnostic (versions 4-6) */
  int32_t rpn_topk;           /* rpn_test_post_nms_topk */
  int32_t result_per_im;      /* 100 */
  int32_t fpn_num_channel;    /* 256 */
  int32_t fc_head_dim;        /* 1024 */
  int32_t precision;          /* 0 = fp16 operands / fp32 accumulate; 1 = split fp16 pair (~fp32 products) */
  int32_t conv_impl;          /* 0 = tensor-core (wgmma) kernel, named "tcgen05" in Python, 1 = CUDA-core cross-check kernel */
  int32_t use_cuda_graph;     /* replay the frame as one CUDA graph */
  float max_size;             /* rounded up to a multiple of 32 by the caller */
  float rpn_min_size, rpn_nms_thres, fastrcnn_nms_iou_thres, result_score_thres;
  float anchor_strides[5], anchor_sizes[5], anchor_ratios[3];
  float bbox_reg_weights[4];
  int32_t accum_chunk;        /* split precision: K-blocks (64 elements) the tensor core accumulates before the
                                 partial sum is folded in with round-to-nearest; 0 = default (1), <0 = never */
  int32_t multi_semantics;    /* 1 = post-processing of Mask_RCNN_FPN_multi (combined_non_max_suppression:
                                 no RPN min-size filter, zero-padded level merge + zero-area drop, no score threshold) */
  int32_t add_mask;           /* --add_mask: mask head on the final boxes (models.py:934-961, 1173-1199; mrcnn_head_dim 256):
                                 ROIAlign 14x14 -> 4 x conv3x3 -> 2x2/2 transposed conv -> conv1x1 -> sigmoid of the box's own
                                 class; results through b2_get_masks */
  int32_t use_gn;             /* --use_gn: GroupNorm (32 groups, statistics per image at run time, nn.py:81-108) instead of
                                 folded BatchNorm in the backbone, and after every FPN lateral / post-hoc conv (nn.py:987-1009) */
  int32_t conv_head_dim;      /* 0 = 2fc head; > 0: --use_conv_frcnn_head with conv_frcnn_head_dim channels (models.py:1110-1125):
                                 4 x conv3x3 + ReLU (+ GroupNorm per ROI with use_gn) -> fc, replacing fc6 / fc7 */
  int32_t use_se;             /* --use_se (--version 6): squeeze-excite in every bottleneck (nn.py:506-519), per image:
                                 relu(conv3 * sigmoid(fc2(relu(fc1(mean_hw(conv3))))) + shortcut), weights
                                 "<block>/fc1/{W,b}" [4*ch, ch/4] and "<block>/fc2/{W,b}" [ch/4, 4*ch] */
  int32_t use_resnext;        /* --use_resnext: ResNeXt 32x4d blocks (nn.py:524-549): conv1 1x1 -> 2*ch, conv2 3x3 2*ch -> 2*ch in
                                 32 groups with SAME padding (weight [3,3,2*ch/32,2*ch]), conv3 1x1 -> 4*ch; no squeeze-excite
                                 (use_se is ignored) */
  int32_t add_relation_nn;    /* --add_relation_nn: relation modules RM_r1 / RM_r2 in the 2fc box head (models.py:1044-1054,
                                 nn.py:115-190): h1 = relu(fc6) + RM_r1(relu(fc6), proposals), h2 = relu(fc7(h1)) +
                                 RM_r2(relu(fc7(h1)), proposals), each image's ROIs attending to its own proposals only;
                                 ignored with conv_head_dim > 0 */
  int32_t use_deformable;     /* --use_deformable: a bottleneck block is deformable when it has stride 2 and is among the last
                                 3 blocks of its group (nn.py:459-521, 568-588): res5 block 0 for R50 / R101 / R152.  Its
                                 conv2 samples conv1's output bilinearly at learned offsets ("<block>/conv2_offset/{W,b}",
                                 [3,3,C,18], [18]) and has no norm and no ReLU.  Each image uses its own offsets.  Ignored
                                 with use_resnext; refused with use_dilations, where the reference's residual sum fails */
} b2_config;

/* Graph options added after b2_config's layout was fixed.  b2_create_ex takes them; b2_create builds the graph with
 * every field 0.  New options are appended here, so a b2_config written against an older header stays valid. */
typedef struct b2_config_ext {
  int32_t use_basic_block;    /* --resnet34 / --resnet18: basic blocks (nn.py:439-456) instead of bottlenecks:
                                 relu(norm(conv2(relu(norm(conv1(x))))) + shortcut), conv1 3x3 at the block's stride and conv2
                                 3x3, both SAME padding and ch_out wide; c2..c5 have 64 / 128 / 256 / 512 channels, and group0
                                 block0's shortcut is the identity.  The block ignores use_dilations, use_deformable and
                                 use_se; use_resnext wins over it (nn.py:864-868) */
} b2_config_ext;

/* Graph options added after b2_config_ext's layout was fixed (one int32, use_basic_block, which callers built against
 * that header pass).  b2_create_ex2 takes them; b2_create_ex builds the graph with every field 0. */
typedef struct b2_config_ext2 {
  int32_t num_partial_classes;     /* --use_partial_classes (models.py:807-828): 0 = off.  Otherwise the box head keeps
                                      only the label logits [0] + partial_class_ids and the box logits of those classes,
                                      in this order, and the post-processing runs over num_partial_classes + 1 classes:
                                      final labels are 1..num_partial_classes, the index into partial_class_ids plus one,
                                      with probabilities from that (num_partial_classes + 1)-way softmax.  The checkpoint
                                      keeps its num_class columns.  The mask head keeps num_class - 1 channels and picks
                                      channel (final label - 1) of them, as the reference does (models.py:934-961).
                                      At most num_class - 1 */
  int32_t partial_class_ids[80];   /* the checkpoint's class ids, each in 1..num_class - 1, no duplicates */
} b2_config_ext2;

/* Graph options added after b2_config_ext2's layout was fixed.  b2_create_ex3 takes them; b2_create_ex2 builds the graph
 * with every field 0. */
typedef struct b2_config_ext3 {
  int32_t use_att_frcnn_head;      /* --use_att_frcnn_head: the attention branch of the class-specific box head
                                      (fastrcnn_2fc_head models.py:1064-1089, batch graph :2682-2707), after fc7 / fc,
                                      the relation modules or the conv head: hidden = hidden + relu(att_trans(sum over the
                                      7x7 bins of the ROIAlign features)), "fastrcnn/att_trans/{W,b}" [256, fc_head_dim].
                                      The reference's 3x3 "fastrcnn/attention" conv has one output channel and a softmax
                                      over that length-1 axis, so its weight is exactly 1 for a finite logit and NaN
                                      otherwise: an ROI with a non-finite feature gets a NaN sum.  The attention weights
                                      are only checked at load (finite, 65536 * sum|W| + |b| below FLT_MAX, so a logit of
                                      finite features stays finite).  Ignored with class_agnostic, whose heads
                                      (models.py:1126-1170) have no attention branch.  Needs fc_head_dim a power of two
                                      from 64 to 2048 */
} b2_config_ext3;

/* Graph options added after b2_config_ext3's layout was fixed.  b2_create_ex4 takes them; b2_create_ex3 builds the graph
 * with every field 0. */
typedef struct b2_config_ext4 {
  int32_t use_small_object_head;   /* main.py --use_small_object_head: the small-object branch of the single-image graph
                                      (models.py:590-692, 845-897), results through b2_get_small_objects.  Per small class:
                                      NMS of its unclipped decoded boxes without a score threshold (at most result_per_im),
                                      ROIAlign 7 -> the head's fc6 / fc7, [optionally + person_object_relation], a [D, 2]
                                      classification; then the head's per-class NMS and top-k over the rebuilt
                                      [K, C + 1] LOGITS.  Every small class must keep the same count K: otherwise the
                                      reference's tf.map_fn fails, and here the status is 1 with K = 0.  Needs batch 1, the
                                      single-image graph and the class-specific 2fc head (refused otherwise, with the
                                      reason); the main outputs do not depend on it */
  int32_t num_small_objects;       /* C, 1 .. min(num_class - 1, 80) */
  int32_t small_object_class_ids[80];   /* the head's class id of each small class, in label order, no duplicates */
  int32_t use_so_association;      /* --use_so_association: hidden += person_object_relation(hidden, boxes, person rows)
                                      (nn.py:194-270), weights "fastrcnn/small_objects/person_object_relation/..." */
  int32_t so_person_class_id;      /* the head's class id of "Person" (with use_so_association) */
  int32_t so_person_topk;          /* --so_person_topk: person boxes kept by their NMS, 1 .. 1024 */
  int32_t use_so_score_thres;      /* --use_so_score_thres: the final NMS keeps logit > result_score_thres only */
} b2_config_ext4;

/* Graph options added after b2_config_ext4's layout was fixed.  b2_create_ex5 takes them; b2_create_ex4 builds the graph
 * with every field 0. */
typedef struct b2_config_ext5 {
  int32_t use_bg_score;            /* main.py --use_bg_score: fastrcnn_predictions (models.py:1263-1270) first drops every
                                      ROI whose argmax over the class probabilities is column 0 (background; ties go to
                                      the lowest column, a NaN never wins), then runs the per-class NMS and top-k over the
                                      kept rows.  As in the reference, a detection's box is then its class's decoded box
                                      of ROI j, j = the selected ROI's rank among the kept rows, not of the selected ROI
                                      itself (models.py:925-930: gather_nd on the unfiltered boxes); its label and
                                      probability are the selected ROI's, and fpn_box_feat / final_masks follow the box.
                                      The small-object branch's final selection filters the same way over its rebuilt
                                      logits (models.py:885-889).  Stages "bg_rank" [B][rpn_topk] and, with the branch,
                                      "so_bg_rank" [result_per_im] hold each row's rank, -1 when dropped.  Ignored with
                                      multi_semantics: the batch graph has no filter (models.py:2924-2976) */
} b2_config_ext5;

const char* b2_last_error(void);
int b2_version(void);

int b2_create(b2_ctx** out, int device, const b2_config* cfg);
/* b2_create with the options of b2_config_ext; ext may be NULL (all 0) */
int b2_create_ex(b2_ctx** out, int device, const b2_config* cfg, const b2_config_ext* ext);
/* b2_create_ex with the options of b2_config_ext2 as well; ext and ext2 may be NULL (all 0).  Refuses, with the reason,
 * partial class ids outside 1..num_class - 1, duplicates and a count above num_class - 1, before touching the device */
int b2_create_ex2(b2_ctx** out, int device, const b2_config* cfg, const b2_config_ext* ext, const b2_config_ext2* ext2);
/* b2_create_ex2 with the options of b2_config_ext3 as well; ext, ext2 and ext3 may be NULL (all 0) */
int b2_create_ex3(b2_ctx** out, int device, const b2_config* cfg, const b2_config_ext* ext, const b2_config_ext2* ext2,
                  const b2_config_ext3* ext3);
/* b2_create_ex3 with the options of b2_config_ext4 as well; ext .. ext4 may be NULL (all 0).  Refuses, with the reason, a
 * small-object configuration the reference cannot build or this engine does not run, before touching the device */
int b2_create_ex4(b2_ctx** out, int device, const b2_config* cfg, const b2_config_ext* ext, const b2_config_ext2* ext2,
                  const b2_config_ext3* ext3, const b2_config_ext4* ext4);
/* b2_create_ex4 with the options of b2_config_ext5 as well; ext .. ext5 may be NULL (all 0) */
int b2_create_ex5(b2_ctx** out, int device, const b2_config* cfg, const b2_config_ext* ext, const b2_config_ext2* ext2,
                  const b2_config_ext3* ext3, const b2_config_ext4* ext4, const b2_config_ext5* ext5);
void b2_destroy(b2_ctx* ctx);

/* Named fp32 host arrays in the reference's Tensorpack-npz naming ("conv0/W",
 * "group1/block0/conv2/bn/mean/EMA", "fpn/lateral_1x1_c2/b", "fastrcnn/fc6/W", ...).
 * BatchNorm is folded, kernels are packed K-major and split into fp16 planes on the device. */
int b2_load_weights(b2_ctx* ctx, const char* const* names, const float* const* data, const int64_t* numel, int n);

/* One pass of the hot path over `batch` frames resident on the device.  All pointers are device
 * pointers; outputs: boxes [B,100,4] x1y1x2y2, probs [B,100], labels [B,100] (1-based), valid [B],
 * box_feat [B*100,C,7,7] fp32 (feat_mode 0) or [B*100,C] mean-pooled (feat_mode 1); any may be NULL.
 * feat_mode 2 / 3 are the TMOT driver's other aggregations (obj_detect_tracking_multi_queuer_tmot.py:511-525): 2 = max over
 * the 7x7 bins [B*100,C], 3 = "spatial" mean over the channels [B*100,49].
 * Asynchronous on the context stream unless `sync` != 0. */
int b2_detect(b2_ctx* ctx, const void* frames_dev, float* boxes, float* probs, int32_t* labels, int32_t* valid,
              float* box_feat, int feat_mode, int sync);
/* Same with host buffers (pinned for full speed): H2D of the frames, the pass, D2H of the results. */
int b2_detect_host(b2_ctx* ctx, const void* frames_host, float* boxes, float* probs, int32_t* labels,
                   int32_t* valid, float* box_feat, int feat_mode);

/* Frame ingest with the resize on the device (SURVEY 8f rank 1).  The reference resizes on the host
 * (frame.astype("float32") -> resizeImage = cv2.resize INTER_LINEAR, nn.py:1540-1560; obj_detect_tracking.py:597-608,
 * enqueuer_thread.py:259-266) and feeds the resized float32 frame.  Here the uint8 source frames [batch, src_h, src_w, 3]
 * (BGR) are uploaded and resized to the context's height x width by a kernel (same bilinear arithmetic, csrc/resize_math.h),
 * then the pass runs as in b2_detect_host.  The context must have input_dtype = 0; the caller picks height / width with
 * get_new_hw (nn.py:1548-1560).  b2_resize_frames runs the resize alone (parity tests), host in / host out. */
int b2_detect_host_resize(b2_ctx* ctx, const uint8_t* frames_u8, int src_h, int src_w, float* boxes, float* probs,
                          int32_t* labels, int32_t* valid, float* box_feat, int feat_mode);
int b2_resize_frames(int device, const uint8_t* frames_u8, int n, int src_h, int src_w, int dst_h, int dst_w,
                     float* out_host);

/* Pipelined ingest for streaming drivers (the queue-fed loop of obj_detect_tracking_multi_queuer.py:386-480):
 * b2_submit_host returns as soon as the upload, the pass and the download of the results are enqueued; b2_wait(slot)
 * blocks until that slot's results are in the caller's buffers.  Two slots: the upload of batch i+1 overlaps the pass
 * of batch i.  Host buffers must stay valid (page-locked for real overlap) until b2_wait returns. */
int b2_submit_host(b2_ctx* ctx, const void* frames_host, float* boxes, float* probs, int32_t* labels, int32_t* valid,
                   float* box_feat, int feat_mode, int slot);
int b2_wait(b2_ctx* ctx, int slot);
/* b2_submit_host for uint8 source frames [batch, src_h, src_w, 3] resized on the device (see b2_detect_host_resize); the
 * source frames must not exceed the network input's float32 byte size (<= 4 source pixels per input pixel). */
int b2_submit_host_resize(b2_ctx* ctx, const uint8_t* frames_u8, int src_h, int src_w, float* boxes, float* probs,
                          int32_t* labels, int32_t* valid, float* box_feat, int feat_mode, int slot);

/* RCNN_FPN_givenbox (models.py:1816-1967, get_model_feat :121-131): final_box_features of GIVEN boxes -- backbone + FPN,
 * ROIAlign 7x7 on the uncropped p2..p5, mean over the bins.  frame_host: one frame of the configured dtype / size (batch 1
 * context), boxes_host [n,4] x1 y1 x2 y2 in frame pixels, feat_host [n, fpn_num_channel]. */
int b2_box_features(b2_ctx* ctx, const void* frame_host, const float* boxes_host, int n, float* feat_host);

/* final_masks of the last pass (needs cfg.add_mask): [batch][result_per_im][28][28] float32 (models.py:958-961; the
 * drivers paste them into the frame with fill_full_mask, obj_detect_tracking.py:719); rows >= valid[b] are zero. */
int b2_get_masks(b2_ctx* ctx, float* masks_host, int64_t capacity_bytes);
/* The small-object branch's outputs of the last pass (use_small_object_head), host buffers: boxes [result_per_im][4]
 * (clipped, resized-image pixels), probs [result_per_im] (the rebuilt LOGITS, models.py:880-897), labels [result_per_im]
 * (1 .. C: index in the small classes + 1), count [1] rows valid, class_counts [C] boxes each small class kept by its
 * NMS, status [1]: 0, or 1 when those counts differ (then count is 0: the reference's graph fails there). */
int b2_get_small_objects(b2_ctx* ctx, float* boxes, float* probs, int32_t* labels, int32_t* count, int32_t* class_counts,
                         int32_t* status);

/* The fetches of main.py --mode forward (main.py:1540-1870) beyond the detections. */
/* fpn_feature (models.py:517-518; --extract_feat, --just_feat): p5 of each image resized to 7 x 7 by TF1's legacy bilinear
 * (align_corners=False, half_pixel_centers=False), feat_host [batch][7][7][fpn_num_channel] float32 NHWC.  The resize
 * samples the p5 of the padded image (23 x 40 at 720 x 1280, 34 x 60 at 1080 x 1920; below 7 it upsamples).
 * frames_host NULL: resizes the p5 of the context's last pass.  Otherwise frames_host [batch][H][W][3] of the context's
 * input dtype are uploaded and only the backbone and FPN run before the resize (with use_cuda_graph, as a graph of their
 * own); such a feature-only pass leaves the detection results, b2_get_* and every stage after the FPN stale: they keep an
 * earlier pass's values.  b2_fpn_feature_launches counts the kernels of that pass, resize included. */
int b2_fpn_feature(b2_ctx* ctx, const void* frames_host, float* feat_host);
int b2_fpn_feature_launches(b2_ctx* ctx);
/* proposal_boxes / proposal_scores of the last pass (models.py:550-558; batch graph 2490-2521), host buffers boxes
 * [batch][rpn_topk][4] x1 y1 x2 y2, scores [batch][rpn_topk], count [batch]: rows >= count[b] are not proposals.  Order:
 * score descending, ties to the lower position in the levels' concatenation (TF's top_k(sorted=False) leaves it open).
 * With multi_semantics zero-area boxes are already dropped (models.py:2516-2521). */
int b2_get_proposals(b2_ctx* ctx, float* boxes, float* scores, int32_t* count);
/* The use_cpu_nms outputs (--no_nms / --save_all_box, models.py:899-916) of image `image` of the last pass, K = its
 * proposal count (*k_out): boxes [num_class - 1][K][4] the decoded, clipped boxes of every class (the class-agnostic
 * head's are the same boxes in every row), probs [num_class - 1][K] the softmax without the background column, rois [K][4]
 * the proposals.  Capacities: (num_class - 1) * rpn_topk * 4, (num_class - 1) * rpn_topk and rpn_topk * 4 floats (with
 * partial classes, their count in place of num_class - 1). */
int b2_get_all_boxes(b2_ctx* ctx, int image, float* boxes, float* probs, float* rois, int32_t* k_out);

/* Mask paste and COCO RLE on the GPU: the drivers' post-processing of final_masks (obj_detect_tracking.py:716-739,
 * obj_detect_imgs.py:501-527), fill_full_mask (nn.py:1565-1584) then pycocotools.mask.encode of the Fortran-ordered frame,
 * bit-exact with cv2.resize (OpenCV 4.13, default dispatch) and pycocotools.  A b2_masks is an encoder bound to one device:
 * its grow-only workspaces and its stream.  boxes_host [n][4] float32 are the final boxes already divided by the resize
 * scale; masks [n][mask_h][mask_w] float32 are host memory, or device memory of the encoder's GPU when masks_on_device.
 * Only 28x28 masks (the mask head's) are accepted.  Each box's patch is placed as fill_full_mask places it; a box whose
 * corner int(box[:2] + 0.5) is below 0, or whose patch NumPy could not broadcast into the frame's slice (the frame edge
 * cuts the slice short, e.g. y1 = H), refuses the call with -2 (message via b2_last_error) before any device work. */
typedef struct b2_masks b2_masks;
int b2_masks_create(b2_masks** out, int device);
void b2_masks_destroy(b2_masks* enc);
/* The full-frame masks fill_full_mask returns: out_host [n][im_h][im_w] uint8 (0 / 1), capacity >= n * im_h * im_w. */
int b2_masks_paste(b2_masks* enc, const float* boxes_host, const float* masks, int masks_on_device, int n, int mask_h,
                   int mask_w, int im_h, int im_w, uint8_t* out_host, int64_t capacity_bytes);
/* The RLE strings pycocotools' rleToString writes (rle["counts"] of the drivers) of the n full-frame masks: offsets_host
 * [n + 1] receives the byte offsets of each string (offsets_host[n] = total bytes, no terminators); the bytes go to
 * bytes_host when capacity >= that total, and stay in the encoder for b2_masks_fetch otherwise. */
int b2_masks_encode(b2_masks* enc, const float* boxes_host, const float* masks, int masks_on_device, int n, int mask_h,
                    int mask_w, int im_h, int im_w, int64_t* offsets_host, char* bytes_host, int64_t capacity);
/* The string bytes of the encoder's last encode (capacity >= its total). */
int b2_masks_fetch(b2_masks* enc, char* bytes_host, int64_t capacity);
/* b2_masks_encode of final_masks rows 0 .. n - 1 of image `image` of the context's last pass (needs cfg.add_mask), read in
 * place on the context's stream: the masks never leave the GPU.  enc must be bound to the context's device; n <=
 * result_per_im. */
int b2_encode_masks(b2_ctx* ctx, b2_masks* enc, int image, const float* boxes_host, int n, int im_h, int im_w,
                    int64_t* offsets_host, char* bytes_host, int64_t capacity);

/* Stage-addressable access for parity tests.  Activations are returned as fp32. */
int b2_stage_shape(b2_ctx* ctx, const char* name, int64_t shape[4], int32_t* dtype /*0 f32, 1 i32*/);
int b2_get_stage(b2_ctx* ctx, const char* name, void* dst_host, int64_t capacity_bytes);
int b2_set_stage(b2_ctx* ctx, const char* name, const void* src_host, int64_t bytes);
/* Run a subset of the pass: bit mask of B2_PHASE_*. */
enum {
  B2_PHASE_BACKBONE = 1, B2_PHASE_FPN = 2, B2_PHASE_RPN_HEAD = 4, B2_PHASE_PROPOSALS = 8,
  B2_PHASE_ROI = 16, B2_PHASE_HEAD_FC = 32, B2_PHASE_POST = 64, B2_PHASE_BOX_FEAT = 128, B2_PHASE_ALL = 255
};
int b2_run_phases(b2_ctx* ctx, int phase_mask);
/* Device time of the last b2_run_phases/b2_detect per phase (ms), measured with CUDA events. */
int b2_phase_times(b2_ctx* ctx, float ms[8]);
int b2_kernel_launches(b2_ctx* ctx);   /* kernels launched by one full pass */
/* Per-launch-group profiling for the roofline report: device ms of every step of the plan (averaged
 * over `reps` eager passes) and a description of each step (algorithmic FLOPs / HBM bytes). */
int b2_num_steps(b2_ctx* ctx);
int b2_profile_steps(b2_ctx* ctx, int reps, float* ms_out, int cap, int* n_out);
int b2_step_info(b2_ctx* ctx, int idx, char* name, int name_cap, double* flops, double* bytes, int* kind);

/* DeepSORT appearance cost: gallery [S,D] rows grouped per track by seg_offsets[T+1], dets [N,D];
 * cost[T,N] = min over the track's rows of (1 - cos).  Host pointers.  Rows are divided by their norm without an eps, as
 * nn_matching: a zero row, or a row with a NaN or inf component, gives NaN, and a NaN among a track's rows makes that
 * track's cost NaN (np.min); the tracker's assignment then refuses the matrix, as the reference's does.  A track with an
 * empty segment gets 3.4e38 for every detection. */
int b2_cosine_cost(int device, const float* gallery, const int32_t* seg_offsets, int T, const float* dets, int N,
                   int D, int precision, float* cost);

/* ---- DeepSORT association loop in native host code (SURVEY 8f rank 2).  Replaces deep_sort/tracker.py:10-138
 * (Tracker.predict / Tracker.update / _match), track.py:19-166, kalman_filter.py:23-232 (float64 state),
 * linear_assignment.py:12-194 (min_cost_matching, matching_cascade, gate_cost_matrix), iou_matching.py:8-81 and the
 * per-track gallery bookkeeping of nn_matching.py:137-154; scipy.optimize.linear_sum_assignment
 * (linear_assignment.py:5,60) is restated natively with SciPy's tie behaviour.  The appearance cost matrix
 * of every cascade level comes from b2_cosine_cost on `device` (one tensor-core GEMM) unless a cost function is
 * installed (tests install the CPU oracle there; there is no built-in CPU path).
 * b2_tracker_create mirrors Tracker(metric, max_iou_distance, max_age, n_init) + NearestNeighborDistanceMetric("cosine",
 * matching_threshold, budget) (tracker.py:40-48, nn_matching.py:120-131; budget <= 0 = None).
 * b2_tracker_update takes the frame's detections: tlwh [n,4] float64, confidence [n] float64 (may be NULL), features
 * [n,feat_dim] float32 (detection.py:27-42).  b2_tracker_get_tracks copies the live tracks in list order (ids, TrackState
 * 1 tentative / 2 confirmed, hits, age, time_since_update, mean [*,8], covariance [*,64]) and returns their number. */
typedef struct b2_tracker b2_tracker;
typedef int (*b2_appearance_cost_fn)(void* user, const float* gallery, const int32_t* seg_offsets, int T,
                                     const float* dets, int N, int D, float* cost);
int b2_tracker_create(b2_tracker** out, int device, double max_iou_distance, int max_age, int n_init,
                      double matching_threshold, int budget, int feat_dim, int precision);
void b2_tracker_destroy(b2_tracker* trk);
int b2_tracker_set_cost_fn(b2_tracker* trk, b2_appearance_cost_fn fn, void* user);
int b2_tracker_predict(b2_tracker* trk);
int b2_tracker_update(b2_tracker* trk, const double* tlwh, const double* confidence, const float* features, int n);
int b2_tracker_num_tracks(b2_tracker* trk);
int b2_tracker_get_tracks(b2_tracker* trk, int cap, int32_t* ids, int32_t* state, int32_t* hits, int32_t* age,
                          int32_t* time_since_update, double* mean, double* cov);
/* scipy.optimize.linear_sum_assignment on a row-major [nr,nc] float64 matrix: writes min(nr,nc) (row, col) pairs sorted by
 * row, returns their number. */
int b2_linear_sum_assignment(const double* cost, int nr, int nc, int32_t* rows, int32_t* cols);
/* application_util/preprocessing.py:6-74 non_max_suppression(boxes tlwh, max_bbox_overlap, scores): writes the kept
 * indices in pick order, returns their number (scores NULL = order by bottom edge, as the reference). */
int b2_track_nms(const double* tlwh, const double* scores, int n, double max_bbox_overlap, int32_t* keep);

/* ---- TMOT / JDE association in native host code (SURVEY 8f rank 4).  Replaces tmot/matching.py:28-109 and the JDETracker loop
 * of tmot/multitracker.py:13-398 (state float64, embeddings float32).  lap.lapjv (lap 0.4.0) and cython_bbox.bbox_overlaps
 * are third-party and absent from the reference tree: restated from their published algorithms (csrc/tmot.cpp header).
 * b2_lapjv              = lap.lapjv(cost, extend_cost=True, cost_limit) as matching.linear_assignment uses it (:28-38) and
 *                         multi_video_reid.py:512: x[nr] / y[nc] = matched column / row or -1, *opt = matched cost sum.
 * b2_tmot_iou_distance  = matching.iou_distance (:57-77): 1 - IoU(+1 pixel convention) of tlbr boxes, out [na,nb].
 * b2_tmot_fuse_motion   = matching.fuse_motion (:97-109): Kalman gate (chi2inv95 of 4 or 2 dof -> inf) and
 *                         cost = lambda * cost + (1 - lambda) * squared Mahalanobis distance, in place on cost [T,N].
 * b2_tmot_embedding_distance = matching.embedding_distance (:80-94): euclidean distance of track / detection embeddings,
 *                         one tensor-core GEMM on `device` (|a|^2 + |b|^2 - 2ab, then sqrt(max(0, .)) with NaN kept, as
 *                         np.maximum), out float64 [T,N]; b2_distance_matrix's range check applies. */
int b2_lapjv(const double* cost, int nr, int nc, double cost_limit, int32_t* x, int32_t* y, double* opt);
int b2_tmot_iou_distance(const double* atlbr, int na, const double* btlbr, int nb, double* out);
int b2_tmot_fuse_motion(const double* means, const double* covs, int T, const double* xyah, int N, double* cost,
                        int only_position, double lambda);
int b2_tmot_embedding_distance(int device, const float* track_feats, int T, const float* det_feats, int N, int D,
                               int precision, double* out);
/* JDETracker(conf_thres, track_max_second_lost, emb_max_dist, iou_max_dist1, iou_max_dist2, emb_smooth_alpha, frame_gap,
 * frame_rate) (multitracker.py:176-204).  Track ids come from a counter shared by every tracker created with the same
 * `share_ids_with` chain (BaseTrack._count is a class attribute, basetrack.py:13,34-37; NULL = own counter).
 * b2_jde_update takes the frame's detections after the pre-tracker NMS: tlwh [n,4] float64, conf [n] float64, features
 * [n,feat_dim] float32 and returns the number of output tracks (tracked and activated, :355).  The embedding distance of
 * the first association comes from b2_distance_matrix on `device` unless a cost function is installed (it then receives
 * one gallery row per track, seg_offsets 0..T, and must write euclidean distances).
 * b2_jde_get_tracks copies list `which` (0 output, 1 tracked_stracks, 2 lost_stracks) in list order; with cap == 0 and
 * ids == NULL it only returns the length. */
typedef struct b2_jde b2_jde;
int b2_jde_create(b2_jde** out, int device, double conf_thres, double track_max_second_lost, double emb_max_dist,
                  double iou_max_dist1, double iou_max_dist2, double emb_smooth_alpha, double frame_gap, double frame_rate,
                  int feat_dim, int precision, b2_jde* share_ids_with);
void b2_jde_destroy(b2_jde* trk);
int b2_jde_set_cost_fn(b2_jde* trk, b2_appearance_cost_fn fn, void* user);
int b2_jde_reset(b2_jde* trk);
/* zeroes only the id counter `trk` shares with its group (multitracker.py:215: reset() of ANY tracker sets BaseTrack._count = 0) */
int b2_jde_reset_ids(b2_jde* trk);
int b2_jde_update(b2_jde* trk, const double* tlwh, const double* conf, const float* features, int n);
int b2_jde_get_tracks(b2_jde* trk, int which, int cap, int32_t* ids, int32_t* state, int32_t* is_activated,
                      int32_t* frame_id, int32_t* start_frame, int32_t* tracklet_len, double* tlwh, double* det_tlwh,
                      double* det_conf, double* score, double* mean, double* cov);

/* ---- ReID embedding: torchreid FeatureExtractor (torchreid/feature_extractor.py:121-252) with osnet_x1_0
 * (torchreid/models/osnet.py:522-534).  b2_reid_create fixes the crop batch; b2_reid_load_weights takes the
 * model's state_dict (torch names, fp32); b2_reid_embed takes host RGB uint8 crops already resized to
 * 256x128 ([n,256,128,3], n <= batch) and returns [n,512] fp32 (ToTensor + Normalize + OSNet eval forward). */
typedef struct b2_reid b2_reid;
int b2_reid_create(b2_reid** out, int device, int batch, int precision);
/* model 0 = osnet_x1_0 as above; model 1 = torchreid's resnet101 (torchreid/models/resnet.py:441-455, the vehicle extractor
 * of single_video_reid.py:410-415): b2_reid_embed then takes crops resized to 128x256 ([n,128,256,3] RGB uint8) and
 * returns [n,2048] (global average pool of layer4, eval mode); state_dict names "conv1.weight", "bn1.*",
 * "layer3.22.conv2.weight", "layer2.0.downsample.0.weight", ... */
int b2_reid_create_model(b2_reid** out, int device, int batch, int precision, int model);
void b2_reid_destroy(b2_reid* ctx);
int b2_reid_load_weights(b2_reid* ctx, const char* const* names, const float* const* data, const int64_t* numel, int n);
int b2_reid_embed(b2_reid* ctx, const uint8_t* crops_host, int n, float* feats_host);
/* Same, with the [n, feat_dim] features left in device memory of the context's GPU (`feats_dev`: e.g. this camera's slice of
 * the gallery buffer the NCCL all-gather of config 5 sends, multi_video_reid.py:448-476) -- a gallery never crosses PCIe. */
int b2_reid_embed_dev(b2_reid* ctx, const uint8_t* crops_host, int n, float* feats_dev);
/* The drivers' whole ReID input step on the GPU (single_video_reid.py:211-227): frames_host is uint8 BGR [nf][h][w][3],
 * boxes_host [n][5] int32 (frame index, x, y, w, h) with 1 <= n <= batch.  Each box is cut out of its frame, turned to RGB
 * and resized to the model's crop size exactly as Pillow's Image.resize(BILINEAR) does, then embedded as b2_reid_embed
 * would embed those crops.  Every box must lie inside its frame with w, h >= 1; a bad box fails the call (b2_last_error)
 * before any device work.  The frames go through a grow-only device buffer the context owns. */
int b2_reid_embed_boxes(b2_reid* ctx, const uint8_t* frames_host, int nf, int h, int w, const int32_t* boxes_host, int n,
                        float* feats_host);
/* Same, with the features left in device memory of the context's GPU, as b2_reid_embed_dev. */
int b2_reid_embed_boxes_dev(b2_reid* ctx, const uint8_t* frames_host, int nf, int h, int w, const int32_t* boxes_host, int n,
                            float* feats_dev);
int b2_reid_feat_dim(b2_reid* ctx);   /* 512 (osnet_x1_0) / 2048 (resnet101) */
int b2_reid_num_launches(b2_reid* ctx);
/* Stage-addressable activation of the last pass as fp32 NHWC (parity tests): "conv1", "maxpool", "conv2.0", ... */
int b2_reid_get_activation(b2_reid* ctx, const char* name, float* dst_host, int64_t capacity_bytes, int64_t shape[4]);

/* ---- EfficientDet (config 3): BiFPN feature network + class/box nets + detection post-processing.
 * Replaces the TF graph of efficientdet/efficientdet_arch.py build_feature_network (:440-505), build_bifpn_layer
 * (:594-682), build_class_and_box_outputs (:343-393) and the wrapper's add_metric_fn_inputs / get_results_tf /
 * own-level ROIAlign box feature (efficientdet_wrapper.py:265-474; anchors.py:399-487). */
typedef struct b2_effdet_config {
  int image_h, image_w;            /* network input size (multiple of 128) */
  int min_level, max_level;        /* 3, 7 */
  int fpn_num_filters, fpn_cell_repeats, box_class_repeats;
  int num_classes, num_scales, num_aspects;
  float aspect_ratios[3][2];       /* (x, y) multipliers, anchors.py:216-257 */
  float anchor_scale;
  int fpn_weight_method;           /* 0 "sum", 1 "fastattn" */
  int backbone_channels[3];        /* channels of the backbone's level 3, 4, 5 endpoints */
  int max_detection_topk;          /* 5000 */
  int result_per_im;               /* 100 */
  float nms_iou_threshold, result_score_thres;
  int precision;                   /* 0 fp16, 1 split (fp32-class) */
  int backbone;                    /* -1: none (b2_effdet_run_features only); 0..7: EfficientNet-b0..b7 trunk
                                    * (efficientdet_arch.py:396-437, backbone/efficientnet_model.py:504-704) */
  int batch;                       /* images per call; 0 or 1: one (b2_effdet_detect / b2_effdet_run_features),
                                    * > 1: b2_effdet_detect_batch, stages gain a leading [batch] */
} b2_effdet_config;
typedef struct b2_effdet b2_effdet;
int b2_effdet_create(b2_effdet** out, const b2_effdet_config* cfg, int device);
void b2_effdet_destroy(b2_effdet* ctx);
/* TF checkpoint variables (names as efficientdet_arch.py creates them, kernels HWIO, fp32) */
int b2_effdet_load_weights(b2_effdet* ctx, const char* const* names, const float* const* data, const int64_t* numel, int n);
/* Backbone endpoints C3/C4/C5 (host NHWC fp32) -> detections: boxes [max][4] x1 y1 x2 y2 scaled by image_scale,
 * scores, classes (1-based), levels, box_feat [max][fpn_num_filters]; *count = number of valid rows. */
int b2_effdet_run_features(b2_effdet* ctx, const float* c3, const float* c4, const float* c5, float image_scale,
                           float* boxes, float* scores, int32_t* classes, int32_t* levels, float* box_feat, int32_t* count);
/* The wrapper's whole per-frame path (efficientdet_wrapper.py:40-111): host BGR uint8 frame [h,w,3] -> build_preprocess
 * (RGB, /255, mean/std, bilinear resize to fit image_h x image_w, zero-pad) -> backbone -> BiFPN -> heads -> detections
 * in frame pixels.  *image_scale_out = image_scale_to_original.  Needs cfg.backbone >= 0. */
int b2_effdet_detect(b2_effdet* ctx, const uint8_t* frame_bgr, int h, int w, float* boxes, float* scores,
                     int32_t* classes, int32_t* levels, float* box_feat, int32_t* count, float* image_scale_out);
/* The same for 1 <= n <= batch independent frames of any sizes (frames[i] is [h[i], w[i], 3]) in one pass of a context
 * created with `batch` images; image i's outputs are bit-identical to b2_effdet_detect(frames[i]) on a batch-1 context.
 * boxes [batch][max][4], scores / classes / levels [batch][max], box_feat [batch][max][fpn_num_filters], counts [batch],
 * image_scales [batch]; rows past counts[i] are zero, blocks i >= n are not written (those images run on the last
 * frame). */
int b2_effdet_detect_batch(b2_effdet* ctx, const uint8_t* const* frames, const int32_t* h, const int32_t* w, int n,
                           float* boxes, float* scores, int32_t* classes, int32_t* levels, float* box_feat, int32_t* counts,
                           float* image_scales);
/* Replays the whole-frame graph the last detect call captured `reps` times on the images as they stand (no host copies);
 * *ms_out = mean milliseconds per replay. */
int b2_effdet_replay(b2_effdet* ctx, int reps, float* ms_out);
/* Stage tensors of the last pass (parity tests): "image", "stem", "block_<i>", "c3".."c5", "fpn3".."fpn7", "cls3".."cls7", "box3".."box7" as fp32 NHWC */
int b2_effdet_get_stage(b2_effdet* ctx, const char* name, float* dst_host, int64_t capacity_bytes, int64_t shape[4]);
/* Post-processing stages: "topk_boxes" [k][4] (ymin xmin ymax xmax, network pixels), "topk_scores" [k], "topk_classes"
 * [k] (int32, 1-based), "topk_levels" [k] (int32), "topk_count" (int32): the candidates in top-k order (logit descending,
 * then flat index); "final_boxes" [max][4] (x1 y1 x2 y2 * image_scale), "final_scores", "final_classes", "final_levels",
 * "final_count" (int32) and "box_feat" [max][fpn_num_filters]: the outputs; "image_scale" (one float).
 * On a context with batch > 1 every stage has shape[0] = batch (image-major), and "topk_count" is the [batch][8] top-k
 * state with each image's count in column 5. */
/* Writes a stage (bytes = its whole stored size) for b2_effdet_run_phases. */
int b2_effdet_set_stage(b2_effdet* ctx, const char* name, const void* src_host, int64_t bytes);
/* Run a subset of the pass eagerly: bit mask of B2_EFFDET_PHASE_*. */
enum { B2_EFFDET_PHASE_BACKBONE = 1, B2_EFFDET_PHASE_FEATURES = 2, B2_EFFDET_PHASE_POST = 4, B2_EFFDET_PHASE_BOX_FEAT = 8 };
int b2_effdet_run_phases(b2_effdet* ctx, int phase_mask);
int b2_effdet_num_launches(b2_effdet* ctx);
/* Per-step CUDA-event timing / description of the pass (same contract as b2_profile_steps / b2_step_info). */
int b2_effdet_profile_steps(b2_effdet* ctx, int reps, float* ms_out, int cap, int* n_out);
int b2_effdet_step_info(b2_effdet* ctx, int idx, char* name, int name_cap, double* flops, double* bytes, int* kind);

/* Distance matrix of torchreid/distance.py:6-80 on the tensor cores: a [na,D], b [nb,D] (host) -> out [na,nb].
 * metric 0 = cosine (1 - a^.b^) with x^ = x / max(|x|, 1e-12) as F.normalize, so a zero row is at distance 1 from every
 * row; 1 = squared euclidean (|a|^2 + |b|^2 - 2 a.b).  A NaN component makes every distance of its row NaN; so does a
 * +-inf one in split precision (fp16 precision may give inf instead).  Metric 1 fails ("outside the fp16-plane range")
 * when a finite component has |x| >= 65520: the fp16 operand plane would hold inf and turn a finite distance into NaN or
 * inf. */
int b2_distance_matrix(int device, const float* a, int na, const float* b, int nb, int D, int metric, int precision,
                       float* out);

/* ---- Multi-camera ReID track-pair costs (BASELINE config 5; multi_video_reid.py:260-324, 486-512).
 * b2_track_pair_cost = compute_feature_dist (:308-324): crop embeddings of camera 1's tracks a [seg_a[N], D] grouped by
 * seg_a[N+1], camera 2's b / seg_b[M+1] (host, float32); out[i][j] = min over the two tracks' crops of the squared
 * euclidean distance (clamped at 0, as sklearn.euclidean_distances) where gate[i][j] != 0 (gate NULL = all pairs), else
 * `fill` (999 in the reference).  One tensor-core GEMM over the concatenated galleries + one segmented-min kernel.
 * A NaN distance in a gated pair's block makes out[i][j] NaN (np.clip and np.min keep NaN); a track with no crops gets
 * `fill`.  A row with a NaN or +-inf component makes all its distances NaN in split precision; a finite component with
 * |x| >= 65520 fails the call ("outside the fp16-plane range"), as in b2_distance_matrix.
 * b2_track_spatial_dist = compute_spatial_dist (:260-305) without the ignore-pairs reset: trajectories as (frame, x, y)
 * rows grouped per track, out[i][j] = mean point distance over common frames (camera-2 frames + frame_offset) if <= tol,
 * else 9999.  Host code, float64. */
int b2_track_pair_cost(int device, const float* a, const int32_t* seg_a, int N, const float* b, const int32_t* seg_b,
                       int M, int D, const uint8_t* gate, float fill, int precision, float* out);
/* The same with the galleries already in device memory.  b_dev may be PEER memory of another GPU of the node (opened with
 * b2_gallery_open): the conversion kernel that builds the GEMM's fp16 operand planes then reads the peer gallery over
 * NVLink directly -- the multi-camera exchange without a staged all-gather copy (one process per GPU; each rank scores its
 * share of the camera pairs against the other ranks' galleries in place).
 * b2_gallery_create uploads a gallery [rows, D] into a cudaMalloc'ed buffer and returns the 64-byte CUDA IPC handle other
 * ranks pass to b2_gallery_open (exchange the handles with any host-side channel, e.g. torch.distributed objects);
 * b2_gallery_close unmaps a peer gallery, b2_gallery_free releases an own one (after the peers have closed it).
 * The call runs on a private non-blocking stream and returns when `out` is complete: device inputs must be complete when it
 * is entered (synchronise the stream / collective that produced them first). */
int b2_track_pair_cost_dev(int device, const float* a_dev, const int32_t* seg_a, int N, const float* b_dev,
                           const int32_t* seg_b, int M, int D, const uint8_t* gate, float fill, int precision, float* out);
int b2_gallery_create(int device, const float* feats_host, int rows, int D, float** dev_out, uint8_t handle_out[64]);
int b2_gallery_open(int device, const uint8_t handle[64], float** peer_out);
int b2_gallery_close(int device, float* peer);
int b2_gallery_free(int device, float* dev);
int b2_track_spatial_dist(const int32_t* frames1, const double* pts1, const int32_t* seg1, int N, const int32_t* frames2,
                          const double* pts2, const int32_t* seg2, int M, int frame_offset, double tol, double* out);

/* ---- Tracklet re-linking within one video (single_video_reid.py:233-306, object_detection_tracking_b200/relink.py).
 * q_dev [seg_q[NQ], D]: the query tracklets' crop features grouped by seg_q[NQ+1]; g_dev / seg_g[NG+1] the gallery
 * tracklets'; both in device memory of `device`.  pairs [P][2] (host) lists (query segment, gallery segment) pairs, in any
 * order and with repeats.  out [P] (host):
 *   method 0 (min_all, :291-299): min over the pair's query rows a and gallery rows b of (|a|^2 + |b|^2) - 2 a.b --
 *     torchreid's squared euclidean, NOT clamped at 0 (b2_track_pair_cost clamps, as sklearn); NaN if any distance of
 *     the block is NaN, as torch.min;
 *   method 1 (avg, :279-290): the same formula on the two segments' float32 means (sum in row order / count).
 * One GEMM of all query rows x all gallery rows (split or fp16 precision, as b2_distance_matrix) and one kernel that
 * reads each pair's block of the products only.  Refused (b2_last_error): offsets that do not start at 0 or decrease, an
 * empty segment (the reference removes tracklets without crops before comparing, :242-261), a pair index outside
 * [0, NQ) x [0, NG), a method other than 0 / 1, and a finite component with |x| >= 65520 ("outside the fp16-plane
 * range").  Runs on a private non-blocking stream and returns when `out` is complete: the device inputs must be complete
 * when it is entered. */
int b2_tracklet_dist_dev(int device, const float* q_dev, const int32_t* seg_q, int NQ, const float* g_dev,
                         const int32_t* seg_g, int NG, int D, const int32_t* pairs, int P, int method, int precision,
                         float* out);

/* Single-op entry used by the kernel parity tests (host pointers, NHWC activations, HWIO kernel). */
int b2_op_conv2d(int device, const float* x, const float* w, const float* bias, const float* res, int B, int H, int W,
                 int Cin, int R, int S, int Cout, int stride, int dil, int pad_t, int pad_b, int pad_l, int pad_r,
                 int relu, int res_shift, int impl, int split, int a_mode, float* out);
/* One conv with the whole conv-kernel contract (the engines' ConvDesc): an input view, a pixel stride, an output placed in
 * a larger buffer, fp32 or plane outputs, an upsampled residual, the epilogue and accumulation options. */
typedef struct b2_conv_view {
  int B, pitch_H, pitch_W, in_ld; /* input buffer x [B][pitch_H][pitch_W][in_ld] */
  int in_H, in_W, Cin;            /* the view: in_H x in_W pixels of Cin channels at the buffer origin (in_ld < Cin:
                                     overlapping windows of consecutive pixels) */
  int R, S, stride, dil, pad_t, pad_b, pad_l, pad_r; /* negative pad_b / pad_r crop */
  int Cout;
  int out_H, out_W, off_h, off_w, ldc; /* output buffer [B][out_H][out_W][ldc]; the Ho x Wo result at (off_h, off_w) */
  int out_f32;                         /* 1: fp32 output, 0: fp16 planes */
  int res_H, res_W, ldr, res_shift;    /* residual [B][res_H][res_W][ldr] read at (y >> res_shift, x >> res_shift) */
  int relu;                            /* 0 none, 1 ReLU, 2 swish */
  int acc_kb, a_mode, force_epi;       /* ConvDesc's accumulation chunk and test knobs (0 / -1 / -1 = the defaults) */
  int impl, split;                     /* impl 0 tensor cores, 1 CUDA cores; split 1 = (hi, lo) planes, 0 = fp16 */
  int b0, nb;                          /* launch over images [b0, b0 + nb) only (nb 0 = all), operands offset by whole
                                          images of their own buffers */
} b2_conv_view;
/* x as above, w HWIO [R][S][Cin][Cout], bias [Cout] and res [B][res_H][res_W][ldr] may be NULL.  out_init
 * [B][out_H][out_W][ldc] is the output buffer's content before the launch (converted to planes for a plane output).  out
 * receives the whole buffer after it (planes joined to fp32); out_hi / out_lo (may be NULL) the raw fp16 planes (out_lo
 * only in split precision); range_flag (may be NULL) the range-monitor word.  Every view, placement and stride is checked
 * against its buffer before any device work. */
int b2_op_conv2d_view(int device, const b2_conv_view* a, const float* x, const float* w, const float* bias,
                      const float* res, const float* out_init, float* out, uint16_t* out_hi, uint16_t* out_lo,
                      uint32_t* range_flag);
/* GroupNorm (32 groups, eps 1e-5) of the view H x W at (off_h, off_w) of x [B][pitch_H][pitch_W][C] (host, fp32, converted to
 * the engine's planes), then + res [B][res_H][res_W][C] read at (y >> res_shift, x >> res_shift) (res may be NULL), then ReLU.
 * per_roi = 1: the box head's one-kernel form (statistics and apply per sample).  out [B][pitch_H][pitch_W][C]: the buffer
 * after the op when in_place, else a zero-initialised output buffer of which only the view is written. */
int b2_op_group_norm(int device, const float* x, const float* res, const float* gamma, const float* beta, int B,
                     int pitch_H, int pitch_W, int C, int H, int W, int off_h, int off_w, int res_H, int res_W, int res_shift,
                     int relu, int per_roi, int split, int in_place, float* out);
/* The SE-ResNet bottleneck's squeeze-excite (nn.py:506-519) as the engine runs it: x [B][H][W][C] (host, fp32, converted to
 * the engine's planes), gate[b] = sigmoid(relu(mean_hw(x[b]) @ w1 + b1) @ w2 + b2) with w1 [C][nr], w2 [nr][C] (nr = C / 16),
 * then out = relu(x * gate[b][c] + res) in place (res [B][H][W][C], may be NULL).  gate_out [B][C] may be NULL. */
int b2_op_squeeze_excite(int device, const float* x, const float* res, const float* w1, const float* b1, const float* w2,
                         const float* b2, int B, int H, int W, int C, int nr, int split, float* out, float* gate_out);
/* Grouped conv (TF conv2d with C / groups input channels per filter, nn.py:352-355) of x [B][H][W][C] with the HWIO
 * weight w [R][S][C/groups][C]: output channel o reads the input channels of its group o / (C/groups).  bias [C] and
 * res [B][Ho][Wo][C] may be NULL; impl 0 = tensor cores (64-channel windows), 1 = CUDA cores (dense block-diagonal). */
int b2_op_group_conv2d(int device, const float* x, const float* w, const float* bias, const float* res, int B, int H, int W,
                       int C, int R, int S, int groups, int stride, int dil, int pad_t, int pad_b, int pad_l, int pad_r,
                       int relu, int impl, int split, float* out);
/* One relation module (relation_network nn.py:115-190, group 16, geo_feat_dim 64) as the box head runs it, per image:
 * h [B][K][D] (host, fp32, converted to the engine's planes), boxes [B][K][4] (x1 y1 x2 y2), count [B] valid rows per
 * image (0..K; rows j >= count[b] take no part), weights geo_emb W [4][64], b [64], geo_conv W [64][16] (the [1,1,64,16]
 * kernel), b [16], query_linear W [D][D], key_linear W [D][D], output_linear W [16*D][D].
 * out [B][K][D] = h + output_linear(softmax_j(log(max(wg, 1e-6)) + q.k / sqrt(D/16)) . h); rows i >= count[b] are h. */
int b2_op_relation(int device, const float* h, const float* boxes, const int32_t* count, const float* geo_emb_w,
                   const float* geo_emb_b, const float* geo_conv_w, const float* geo_conv_b, const float* query_w,
                   const float* key_w, const float* output_w, int B, int K, int D, int split, float* out);
/* The attention box head's pool (use_att_frcnn_head) as the engine runs it: x [M][49][C] (host, fp32, converted to the
 * engine's planes, the ROIAlign row order), out [M][C] fp32 = the sum over the 49 bins, in bin order, read back from its
 * planes; a row whose 49 x C values are not all finite is all NaN.  C a multiple of 8 up to 8192; the planes hold sums up
 * to 65504 in magnitude (the engine's pass fails beyond that, as for every plane output). */
int b2_op_att_pool(int device, const float* x, int M, int C, int split, float* out);
/* person_object_relation (nn.py:194-270, use_so_association) as the engine runs it: query rows h [K][D] with boxes [K][4],
 * key rows ref [R][D] with boxes ref_boxes [R][4] (host, fp32; the rows are converted to the engine's planes), the
 * module's weights (geo_emb W [4][64], b [64], geo_conv W [64][16], b [16], query / key W [D][D], output W [16D][D]).
 * out [K][D] = h + output_linear(P . ref), P the softmax over the R key rows; read back from its planes.  D a multiple of
 * 64, 1 <= R <= 1024. */
int b2_op_so_attend(int device, const float* h, const float* boxes, int K, const float* ref, const float* ref_boxes, int R,
                    const float* geo_emb_w, const float* geo_emb_b, const float* geo_conv_w, const float* geo_conv_b,
                    const float* query_w, const float* key_w, const float* output_w, int D, int split, float* out);
/* The mask head (models.py:934-961, 1173-1199) as the engine runs it, each layer into its own buffer: feats p2..p5 one
 * after the other, level l [B][pitch_H][pitch_W][C] (host, fp32, converted to the engine's planes) with level_hw[4 l ..
 * 4 l + 3] = (pitch_H, pitch_W, H, W), (H, W) the crop ROIAlign sees, and strides[l]; boxes [B][R][4] (x1, y1, x2, y2),
 * count [B] in [0, R] and labels [B][R] (1 .. num_class - 1 below the count); the weights maskrcnn/fcn0..3/{W,b},
 * maskrcnn/deconv/{W,b} and maskrcnn/conv/{W,b} under their checkpoint names (as b2_load_weights).  Outputs (each may be
 * NULL but masks): roi [M][14][14][C] (M = B R) the ROIAlign 14 rows, fcn [4][M][14][14][C], up [M][14][14][4C] the
 * deconv's (tap, channel) rows, each joined to fp32 and as raw planes (the lo planes unwritten in fp16 precision);
 * logits [M * 784][ld] (ld = num_class - 1 rounded up to 16) the class conv; masks [B][R][28][28], 0 beyond the count.
 * With logits_in ([M * 784][ld]) the own-class sigmoid alone runs on it, and feats, level_hw, strides, boxes and the
 * weights may be NULL.  C must be 256.  Sizes, counts and labels are checked before any device work. */
int b2_op_mask_head(int device, const float* feats, const int32_t* level_hw, const float* strides, int C, int B, int R,
                    const float* boxes, const int32_t* count, const int32_t* labels, int num_class,
                    const char* const* names, const float* const* data, const int64_t* numel, int n,
                    const float* logits_in, int split, float* roi, uint16_t* roi_hi, uint16_t* roi_lo, float* fcn,
                    uint16_t* fcn_hi, uint16_t* fcn_lo, float* up, uint16_t* up_hi, uint16_t* up_lo, float* logits,
                    float* masks);
/* The deformable conv's bilinear sampler (deformable_conv2d nn.py:1642-1712, deformable_helper.py:42-137) as the engine runs
 * it: x [B][H][W][C] (host, fp32, converted to the engine's planes), offsets [B][ceil(H/2)][ceil(W/2)][18] (channel 2k the
 * y and 2k+1 the x offset of tap k, per image).  out [B][ceil(H/2)][ceil(W/2)][9][C]: the sampled operand read back from
 * its planes.  C a multiple of 64. */
int b2_op_deform_sample(int device, const float* x, const float* offsets, int B, int H, int W, int C, int split, float* out);
/* The whole deformable conv2 as the engine runs it: offsets = 3x3 stride-2 conv of x with offset_w [3][3][C][18] and
 * offset_b [18] (pads 1 top / left), the sampler, then the conv w [3][3][C][Cout] over the sampled operand with no bias,
 * norm or activation; Cout == C.  out [B][ceil(H/2)][ceil(W/2)][Cout]; offsets_out (may be NULL)
 * [B][ceil(H/2)][ceil(W/2)][18].
 * impl 0 = tensor cores, 1 = CUDA cores (both for the offset conv and conv2). */
int b2_op_deform_conv2d(int device, const float* x, const float* offset_w, const float* offset_b, const float* w, int B,
                        int H, int W, int C, int Cout, int impl, int split, float* out, float* offsets_out);

/* The element-wise and reduction kernels around the GEMMs, one at a time.  Activations are host fp32 converted to the
 * engine's planes; a plane output is returned joined to fp32 in `out` and, where out_hi / out_lo are not NULL, as its raw
 * fp16 planes (out_lo only in split precision).  Every size is checked before any device work.
 *
 * Depthwise conv of x [B][H][W][C] (C a multiple of 8) with w [K*K][C] (BatchNorm scale folded) and bias [C] into
 * out [B][Ho][Wo][C].  impl 0, EfficientNet's strip kernel: B = 1, K 3 or 5, stride 1 or 2, output (y, x) reads input
 * (y * stride - pad_t + r, x * stride - pad_l + s), zero outside the map; bias may be NULL; act 0 none, 2 swish.
 * impl 1, OSNet's LightConv3x3 depthwise half: K = 3, stride 1, pad 1, Ho = H, Wo = W, bias given, act 1 (ReLU). */
int b2_op_depthwise(int device, const float* x, const float* w, const float* bias, int B, int H, int W, int C, int K,
                    int stride, int pad_t, int pad_l, int Ho, int Wo, int act, int impl, int split, float* out,
                    uint16_t* out_hi, uint16_t* out_lo);
/* A pool of x [B][H][W][C] (C a multiple of 8).  kind 0: the detector's and the ReID stems' 3x3 stride-2 max-pool, window
 * rows 2y - 1 .. 2y + 1 (columns alike) clipped to the map, out [B][Ho][Wo][C] with the caller's Ho <= ceil(H / 2),
 * Wo <= ceil(W / 2); the running maximum starts from 0, so it is the max-pool only of inputs >= 0 (every caller feeds it
 * post-ReLU data), and it keeps the (hi, lo) pair of the element with the largest joined value.  kind 1: AvgPool2d(2),
 * out [B][H / 2][W / 2][C].  kind 2: the global average pool, C a multiple of 64, out [B][out_ld] fp32 holding the
 * buffer's content before the call (columns >= C keep it); out_hi / out_lo unused. */
int b2_op_pool(int device, const float* x, int kind, int B, int H, int W, int C, int Ho, int Wo, int out_ld, int split,
               float* out, uint16_t* out_hi, uint16_t* out_lo);
/* One BiFPN node combine: n_in (1 to 3) inputs one after the other in x, input i [B][hw[2i]][hw[2i+1]][C], each resampled
 * to Ho x Wo as the EfficientDet engine does (same size: read as is; 2x larger: 3x3 stride-2 max-pool with TF SAME
 * padding; half the size: nearest 2x upsampling), then node = sum_i x_i * relu(w_i) / (sum_i relu(w_i) + 1e-4) with the
 * raw fastattn weights (weights [n_in], or NULL for the plain sum), then x * sigmoid(x) when swish.  out [B][Ho][Wo][C];
 * resample [n_in][3] (may be NULL) receives each input's (mode 0 / 1 / 2, pad_t, pad_l). */
int b2_op_bifpn_combine(int device, const float* x, const int32_t* hw, const float* weights, int n_in, int B, int Ho,
                        int Wo, int C, int swish, int split, float* out, uint16_t* out_hi, uint16_t* out_lo,
                        int32_t* resample);
/* MBConv's squeeze-excite: x [B][HW][Cpad] with channels [0, Creal) live, w1 [Creal][nr], b1 [nr], w2 [nr][Creal],
 * b2 [Creal]; gate [B][Cpad] = sigmoid(swish(mean(x) @ w1 + b1) @ w2 + b2), 0 in columns >= Creal.  With w, the
 * projection's fp32 master weight [rows][Cpad] (B = 1), the folded weight w[o][c] * gate[c] is returned as planes in
 * w_hi / w_lo and joined in w_out (all [rows][Cpad]); with w NULL only the gate is computed. */
int b2_op_mbconv_se(int device, const float* x, const float* w1, const float* b1, const float* w2, const float* b2,
                    const float* w, int B, int HW, int Cpad, int Creal, int nr, int rows, int split, float* gate,
                    float* w_out, uint16_t* w_hi, uint16_t* w_lo);
/* OSNet's ChannelGate over an OSBlock's four streams and their gated sum: s [4][B][HW][C] (C a multiple of 64, channels
 * [0, Creal) live), w1 [Cr][Creal], b1 [Cr], w2 [Creal][Cr], b2 [Creal]; gates [B][4][C] = sigmoid(relu(gap(s_k[b]) @ w1^T
 * + b1) @ w2^T + b2), 0 in columns >= Creal; out [B][HW][C] = sum_k gates[b][k] * s_k[b].  gates_in [B][4][C] (may be
 * NULL) replaces the computed gates, so that the gated sum runs alone; gates_out (may be NULL) receives the gates used. */
int b2_op_channel_gate(int device, const float* s, const float* w1, const float* b1, const float* w2, const float* b2,
                       const float* gates_in, int B, int HW, int C, int Creal, int Cr, int split, float* gates_out,
                       float* out, uint16_t* out_hi, uint16_t* out_lo);
/* EfficientNet's stem operand: img [H][W][3] fp32 -> out [Ho][Wo][64], column (r * 3 + s) * 3 + c of pixel (y, x) =
 * img[2y - pad_t + r][2x - pad_l + s][c] (0 outside the image), columns 27..63 zero. */
int b2_op_stem_im2col(int device, const float* img, int H, int W, int Ho, int Wo, int pad_t, int pad_l, int split,
                      float* out, uint16_t* out_hi, uint16_t* out_lo);
/* The ResNet stems' operand packs: frames img [B][H][W][3] (uint8 when is_u8, else float32) normalised and packed into
 * out [B][Hu][Wu][L] with P the normalised frame, zero outside it:
 *   layout 0, the detector (L = 16, any float32 allowed): lane ry*6 + sx*3 + c of pixel (y, x) = P[2y + ry - 3][2x + sx - 3][c],
 *     lanes 12..15 zero; P = (x * (1/255) - mean) / std with BGR constants;
 *   layout 1, the ReID engines (L = 64, uint8 only): lane s*12 + ry*6 + sx*3 + c of pixel (y, q) =
 *     P[2y + ry - 3][2(q + s) + sx - 3][c], lanes 48..63 zero; P = (x / 255 - mean) / std with RGB constants.
 * out is the operand joined to fp32, out_hi / out_lo (may be NULL; out_lo unwritten in fp16 precision) its raw planes. */
int b2_op_stem_pack(int device, const void* img, int is_u8, int B, int H, int W, int layout, int Hu, int Wu, int split,
                    float* out, uint16_t* out_hi, uint16_t* out_lo);
/* The ReID crop resize of b2_reid_embed_boxes alone: frames [nf][h][w][3] uint8 BGR and boxes [n][5] int32 (frame, x, y,
 * w, h; host memory, checked as there) -> out [n][out_h][out_w][3] uint8 RGB, each box resized as Pillow's
 * Image.resize((out_w, out_h), BILINEAR); 1 <= out_w <= 256. */
int b2_op_reid_crop_resize(int device, const uint8_t* frames, int nf, int h, int w, const int32_t* boxes, int n, int out_h,
                           int out_w, uint8_t* out);

/* The distance kernels of b2_cosine_cost, b2_distance_matrix, b2_track_pair_cost and b2_tmot_embedding_distance, one at a
 * time.  b2_op_distance_operand converts x [rows][D] (host fp32) into the GEMM's operand planes out_hi / out_lo
 * [rows][ld] (raw fp16, ld >= D, columns >= D zero): normalize != 0, cosine_normalize_rows, x / max(|x|, eps) with the
 * norm summed in fp32; normalize == 0, rows_to_planes, x itself, with sqnorm [rows] = sum x^2 in fp32 and range_flag = 1
 * when a finite component rounds to an fp16 inf (sqnorm and range_flag may be NULL, and are not written when
 * normalize != 0). */
int b2_op_distance_operand(int device, const float* x, int rows, int D, int ld, int normalize, float eps, uint16_t* out_hi,
                           uint16_t* out_lo, float* sqnorm, uint32_t* range_flag);
/* b2_op_distance_epilogue runs one epilogue on host products dots [rows][ld] (ld >= cols), every step one IEEE fp32 op:
 * kind 0: out [rows][cols] = 1 - dots; kind 1: out = (na2[i] + nb2[j]) - 2 dots[i][j], na2 [rows], nb2 [cols];
 * kind 2: out [n_a][cols] = min over rows s in [seg_a[t], seg_a[t+1]) of 1 - dots[s][n] (NaN if any is NaN, 3.4e38 for
 * an empty segment); kind 3: out [n_a][n_b] = min over the block (rows of segment i of seg_a, columns of segment j of
 * seg_b) of max(0, kind 1's value), NaN if any is NaN, `fill` where gate[i][j] == 0 (gate [n_a][n_b] may be NULL) or a
 * segment is empty.  Offsets are checked against rows / cols before any device work. */
int b2_op_distance_epilogue(int device, int kind, const float* dots, int rows, int cols, int ld, const float* na2,
                            const float* nb2, const int32_t* seg_a, int n_a, const int32_t* seg_b, int n_b,
                            const uint8_t* gate, float fill, float* out);

#ifdef __cplusplus
}
#endif
#endif  /* B200DET_H_ */
