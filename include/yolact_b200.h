/*
 * yolact_b200.h -- C ABI of libyolact_b200.so: the H100-native (sm_90a) YOLACT hot path.
 *
 * The reference (feiyuhuahuo/Yolact_minimal @ d920c05) is pure Python/PyTorch plus one Cython
 * file; it has no FFI.  Its drop-in boundary is three Python import points (SURVEY.md 8(b)):
 *     modules/yolact.py:141-164      Yolact.forward            -> yb_net_forward / yb_net_detect_host
 *     utils/output_utils.py:126-163  nms (+ fast_nms :11-43, traditional_nms :84-123)
 *                                                               -> yb_detect
 *     utils/output_utils.py:200-233  after_nms (+ box_utils.py:147-168 crop)
 *                                                               -> yb_mask_assemble
 *     cython_nms.pyx:24-74           nms(dets, thresh)          -> yb_hard_nms / yb_hard_nms_host
 * The Python package yolact_minimal_b200 mirrors those import points and binds this library
 * through ctypes (INTEGRATION.md shows the stubs).  Signatures use plain pointers and sizes only.
 *
 * Conventions
 *   - every entry point returns a yb_status (0 = ok, <0 = error); yb_last_error() returns a
 *     thread-local message for the last failure.  Nothing here falls back to a CPU path.
 *   - pointers are DEVICE pointers unless the function name ends in _host.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Device entry
 *     points are asynchronous on that stream; *_host entry points synchronise before returning.
 *   - all tensors are dense, row-major, float32 unless stated.
 */
#ifndef YOLACT_B200_H_
#define YOLACT_B200_H_

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define YB_API __attribute__((visibility("default")))
#else
#define YB_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  YB_OK = 0,
  YB_ERR_INVALID = -1,      /* bad argument */
  YB_ERR_CUDA = -2,         /* CUDA runtime / driver failure */
  YB_ERR_UNSUPPORTED = -3,  /* shape or option outside what the kernels are built for */
  YB_ERR_STATE = -4         /* call order (e.g. forward before finalize) */
} yb_status;

#define YB_VERSION 100

YB_API int yb_version(void);
YB_API const char* yb_last_error(void);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
YB_API uint64_t yb_launch_count(void);
/* sm_count / compute capability of the current device */
YB_API int yb_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ------------------------------------------------------------------------------------------
 * Post-process: score filter + SSD box decode + Fast-NMS (or per-class greedy NMS) + top-k.
 * Replaces utils/output_utils.py:126-163 nms(), :11-43 fast_nms(), :84-123 traditional_nms().
 * Batched over images (the reference is batch-1 only: output_utils.py:127-130).
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  float score_thr;    /* cfg.nms_score_thre  (config.py:122)  keep anchor iff max_fg_score >  thr */
  float iou_thr;      /* cfg.nms_iou_thre    (config.py:123)  Fast: keep iff max IoU <= thr; hard: suppress iff >= thr */
  int top_k;          /* cfg.top_k           (config.py:124)  <= 256 */
  int max_det;        /* cfg.max_detections  (config.py:125)  <= 256 */
  int num_classes;    /* incl. background column 0 (81) */
  int coef_dim;       /* 32 */
  int traditional;    /* cfg.traditional_nms: 0 = Fast-NMS, 1 = per-class greedy NMS in pixel coords */
  float img_size;     /* cfg.img_size, only used when traditional != 0 */
  int no_clip;        /* 0: clip decoded boxes to [0,1] (nms(), output_utils.py:153); 1: no clip -- the ONNX/TRT callers' nms_numpy (:186-190) */
} yb_detect_params;

YB_API size_t yb_detect_workspace_bytes(int batch, int num_anchors, const yb_detect_params* p);

/* cls [B,A,C] post-softmax, box [B,A,4], coef [B,A,K], anchors [A,4] (cx,cy,w,h).
 * Outputs (all [B,max_det,...], rows >= out_count[b] are zero-filled):
 *   out_count [B] int32, out_class [B,max_det] int32 (0-based fg class),
 *   out_anchor [B,max_det] int32, out_score [B,max_det], out_box [B,max_det,4] corner form in
 *   [0,1], out_coef [B,max_det,K] (may be NULL). */
YB_API int yb_detect(const float* cls, const float* box, const float* coef, const float* anchors,
              int batch, int num_anchors, const yb_detect_params* p,
              void* workspace, size_t workspace_bytes,
              int32_t* out_count, int32_t* out_class, int32_t* out_anchor,
              float* out_score, float* out_box, float* out_coef, void* stream);

/* Same call with HOST buffers: allocates/copies/synchronises internally (the nms() a Python
 * or C caller with numpy arrays would make).  */
YB_API int yb_detect_host(const float* cls, const float* box, const float* coef, const float* anchors,
                   int batch, int num_anchors, const yb_detect_params* p,
                   int32_t* out_count, int32_t* out_class, int32_t* out_anchor,
                   float* out_score, float* out_box, float* out_coef);

/* ------------------------------------------------------------------------------------------
 * Greedy hard NMS -- replaces cython_nms.pyx:24-74 nms(dets, thresh).
 * dets [n,5] (x1,y1,x2,y2,score) in pixels; '+1' areas; suppress iff ovr >= thresh.
 * out_keep [n] uint8 flags in ORIGINAL order (the reference returns np.where(flag)[0]).
 * ---------------------------------------------------------------------------------------- */
YB_API int yb_hard_nms(const float* dets, int n, float thresh, uint8_t* out_keep, void* stream);
YB_API int yb_hard_nms_host(const float* dets, int n, float thresh, uint8_t* out_keep);

/* ------------------------------------------------------------------------------------------
 * Mask assembly -- replaces utils/output_utils.py:217-231 (after_nms) + box_utils.py:147-168.
 *   masks = sigmoid(proto[P,P,K] @ coef[d,K]^T); crop to box (+1 px pad); bilinear resize to
 *   max(h,w)^2 (align_corners=False); > 0.5; slice to h x w; boxes*max(h,w) -> int32 (trunc).
 * proto [P,P,K], coef [d,K], box [d,4]; out_mask [d,img_h,img_w] (mask_f32 = 0: uint8 0/1; 1: float32 0/1 -- the reference's
 * dtype; 2: BIT-PACKED uint32 words [d,img_h,ceil(img_w/32)], pixel x = bit x & 31 of word x >> 5); out_box_px [d,4] int32.
 * workspace: d*P*P floats.
 * ---------------------------------------------------------------------------------------- */
YB_API size_t yb_mask_workspace_bytes(int num_det, int proto_size);
YB_API int yb_mask_assemble(const float* proto, const float* coef, const float* box, int num_det,
                     int proto_size, int coef_dim, int img_h, int img_w, int crop, int mask_f32,
                     void* workspace, size_t workspace_bytes,
                     void* out_mask, int32_t* out_box_px, void* stream);

/* ------------------------------------------------------------------------------------------
 * Mask output stage (SURVEY.md 8(f) rank 2) -- what the reference's evaluation loop does with the masks after after_nms:
 *   yb_pack_mask_bits   {0,1} masks [n,h,w] (uint8, or float32 when is_f32) -> packed words [n,h,ceil(w/32)]
 *   yb_mask_iou_bits    utils/box_utils.py:189-200 mask_iou on packed masks: out [n,m] = |a&b| / (|a| + |b| - |a&b|); `words` = words per mask
 *   yb_box_iou          utils/box_utils.py:8-37 box_iou for [n,4] x [m,4] corner boxes -> [n,m]
 *   yb_mask_rle         the run lengths of pycocotools.mask.encode(np.asfortranarray(mask)) (utils/common_utils.py:88-96): column-major
 *                       scan, first count = leading zeros (possibly 0).  counts [n,max_runs] uint32, nruns [n] (negative = -needed
 *                       when max_runs is too small).  The ASCII compression of the counts is host work (utils/mask_utils.py).
 * ---------------------------------------------------------------------------------------- */
YB_API int yb_pack_mask_bits(const void* masks, int is_f32, int n, int h, int w, uint32_t* out, void* stream);
YB_API int yb_mask_iou_bits(const uint32_t* a, int n, const uint32_t* b, int m, int64_t words, float* out, void* stream);
YB_API int yb_box_iou(const float* a, int n, const float* b, int m, float* out, void* stream);
YB_API int yb_mask_rle(const uint32_t* bits, int n, int h, int w, uint32_t* counts, int max_runs, int32_t* nruns, void* stream);

/* ------------------------------------------------------------------------------------------
 * Evaluation: box and mask mAP -- replaces utils/common_utils.py:107-255 (APDataObject, prep_metrics, calc_map) as eval.py:35-69
 * and :106 drive them, batched over images.  Results equal the reference's float64 values bit for bit:
 *   yb_eval_match  per image: box IoU (scaled gt vs int pixel boxes, fp32) and popcount mask IoU for same-class pairs, then
 *                  prep_metrics' greedy matching for every (IoU type, threshold): detections of a class in their given order,
 *                  each takes the unused gt of its class with the largest IoU > thr (compared in double; ties -> earliest gt;
 *                  NaN never matches).  Appends one record (score, class, tp bits) per detection at the image's position in
 *                  the caller's record buffers (running count + exclusive prefix of earlier images' counts: no host sync) and
 *                  adds the image's per-class gt counts and "seen" flags.  Images with count == 0 contribute nothing
 *                  (eval.py:53 skips them before prep_metrics, so their gts are never counted).
 *                  tp bit (type * num_thr + t): type 0 = box, 1 = mask.
 *  yb_eval_ap      APDataObject.get_ap for every (type, threshold, class): stable sort of the records by (class, descending
 *                  score; ties keep record order = image order, then detection order), precision / recall in double, the
 *                  running max from the right, np.searchsorted(recalls, x / 100, 'left') at 101 points, their sum in order with
 *                  the Neumaier compensation of Python's sum() (CPython >= 3.12) / 101;
 *                  0 when the class has no gt.  ap [2][num_thr][num_classes] float64, nonempty [num_classes] (1 iff the class
 *                  occurred among the detections or gts of an evaluated image: !APDataObject.is_empty()).
 * Inputs of yb_eval_match (DEVICE pointers; batch B, max_det D):
 *   count [B], cls [B,D] (0-based class), score [B,D]: detect_batched's record layout; box_px [B,D,4] int32 pixel boxes (after_nms)
 *   det_masks: packed masks (yb_pack_mask_bits layout) of all images back to back; image b owns words det_mask_off[b] ..
 *              det_mask_off[b+1] (int64 [B+1]), at least count[b] masks of img_hw[b] = (h, w) (int32 [B,2]); det_mask_words =
 *              words in det_masks
 *   gt [total_gt,5] (x1,y1,x2,y2 in [0,1], class) and gt_offset [B+1] as in yb_losses; gt_masks / gt_mask_off / gt_mask_words
 *              likewise for the packed gt masks, exactly one per gt row (gt row r of image b is mask r - gt_offset[b] of the image)
 *   records: rec_score / rec_cls / rec_tp [capacity]; classes outside [0, num_classes) are stored as -1 and never counted
 *   state [yb_eval_state_bytes]: zeroed by the caller before the first batch.  Bytes 0-7: records appended so far (uint64);
 *              bytes 12-15: error flags (bit 0: capacity exceeded, bit 1: an image's gt or mask ranges lie outside the buffers
 *              or do not match its geometry; such an image's records are stored with class -1).
 * ---------------------------------------------------------------------------------------- */
#define YB_EVAL_MAX_THR 16
typedef struct {
  int num_classes;                 /* len(cfg.class_names) */
  int num_thr;                     /* len(iou_thres), 1 .. YB_EVAL_MAX_THR (eval.py uses 10) */
  double thr[YB_EVAL_MAX_THR];     /* iou_thres (eval.py:24): x / 100 */
} yb_eval_params;

YB_API size_t yb_eval_state_bytes(const yb_eval_params* p);
YB_API size_t yb_eval_match_workspace_bytes(int batch, int max_det, int64_t total_gt, const yb_eval_params* p);
YB_API size_t yb_eval_ap_workspace_bytes(int64_t num_records, const yb_eval_params* p);
YB_API int yb_eval_match(const yb_eval_params* p, int batch, int max_det, const int32_t* count, const int32_t* cls, const float* score,
                         const int32_t* box_px, const uint32_t* det_masks, const int64_t* det_mask_off, int64_t det_mask_words,
                         const int32_t* img_hw, const float* gt, const int32_t* gt_offset, int64_t total_gt, const uint32_t* gt_masks,
                         const int64_t* gt_mask_off, int64_t gt_mask_words, float* rec_score, int32_t* rec_cls, uint32_t* rec_tp,
                         int64_t capacity, void* state, void* workspace, size_t workspace_bytes, void* stream);
/* num_records: an upper bound of the records appended (the records beyond the state's count are ignored) */
YB_API int yb_eval_ap(const yb_eval_params* p, const float* rec_score, const int32_t* rec_cls, const uint32_t* rec_tp, int64_t num_records,
                      const void* state, void* workspace, size_t workspace_bytes, double* ap, uint8_t* nonempty, void* stream);

/* ------------------------------------------------------------------------------------------
 * Pre-process -- replaces utils/augmentations.py:219-227 val_aug(img, val_size) (SURVEY.md 8(f) #1):
 * uint8 BGR HWC image [h,w,3] (device) -> float32 RGB CHW [3,S,S] (device): pad to square at the
 * top-left with the BGR mean, bilinear resize (OpenCV INTER_LINEAR coordinates), (x-mean)/std.
 * ---------------------------------------------------------------------------------------- */
YB_API int yb_val_aug(const uint8_t* img_bgr, int h, int w, int img_size, float* out, void* stream);

/* ------------------------------------------------------------------------------------------
 * Network: ResNet-50/101 + FPN + ProtoNet + prediction heads (modules/resnet.py,
 * modules/yolact.py:12-164), eval forward.  Weights are handed over by their reference
 * state-dict names (SURVEY.md App. C); BatchNorm is folded at finalize time.
 * ---------------------------------------------------------------------------------------- */
typedef struct yb_net yb_net;

/* FP32: CUDA-core fp32 (parity mode).  BF16 / FP16: 16-bit activations and weights on the
 * wgmma tensor cores with fp32 accumulation (FP16 has TF32's 10-bit mantissa: the accuracy
 * of the reference's own GPU path; BF16 has 8 bits). */
typedef enum { YB_PREC_FP32 = 0, YB_PREC_BF16 = 1, YB_PREC_FP16 = 2 } yb_precision;

typedef struct {
  int depth;          /* 50 or 101 */
  int img_size;       /* square input side, any value >= 64 (550 and 400 are fine) */
  int num_classes;    /* incl. background (81) */
  int num_ratios;     /* len(cfg.aspect_ratios) = 3 */
  int coef_dim;       /* 32 */
} yb_net_config;

YB_API int yb_net_create(const yb_net_config* cfg, yb_net** out);
YB_API void yb_net_destroy(yb_net* net);
/* number of parameter tensors the net expects, and the name / element count of the i-th */
YB_API int yb_net_num_params(const yb_net* net);
YB_API int yb_net_param_info(const yb_net* net, int i, const char** name, int64_t* count);
/* data: HOST float32 array with `count` elements, reference layout (conv: [Cout,Cin,kh,kw]) */
YB_API int yb_net_set_param(yb_net* net, const char* name, const float* data, int64_t count);
/* folds BN, packs weights, allocates the activation arena for up to max_batch images */
YB_API int yb_net_finalize(yb_net* net, int max_batch, int precision);
YB_API int yb_net_num_anchors(const yb_net* net);
YB_API int yb_net_proto_size(const yb_net* net);
/* anchors [A,4] float32 (cx,cy,w,h), computed in float64 and rounded once (box_utils.py:86-101) */
YB_API int yb_net_anchors_host(const yb_net* net, float* out);
YB_API const float* yb_net_anchors_device(const yb_net* net);
/* Replace the built-in anchor table (COCO scales int(S/544*{24,48,96,192,384}), ratios {1, 1/2, 2}: config.py:80-81) by the
 * caller's [A,4] (cx,cy,w,h) float32 HOST table -- custom cfg.scales / cfg.aspect_ratios (e.g. res50_pascal, config.py:196).
 * num_anchors must equal yb_net_num_anchors(); callable before or after finalize. */
YB_API int yb_net_set_anchors(yb_net* net, const float* anchors_host, int num_anchors);

/* img [B,3,S,S] NCHW float32 (device).  Outputs (device): cls [B,A,C] softmaxed, box [B,A,4],
 * coef [B,A,K] (tanh), proto [B,P,P,K] (relu, NHWC) -- Yolact.forward's eval 4-tuple. */
YB_API int yb_net_forward(yb_net* net, const float* img, int batch,
                   float* cls, float* box, float* coef, float* proto, void* stream);

/* Debug/parity taps: copy a named intermediate activation ("c3","c4","c5","p3".."p7") of the
 * last forward into out as NCHW float32 [B,C,H,W] (device). */
YB_API int yb_net_read_activation(yb_net* net, const char* name, int batch, float* out, int64_t out_count,
                           int* C, int* H, int* W, void* stream);

/* Per-kernel timing of yb_net_forward with CUDA events on the launching stream (bench.py's
 * roofline numbers).  While enabled every forward records one event per layer; yb_net_profile
 * synchronises, aggregates the layers by kernel ("conv_tc", "conv_simt", "stem", ...) over all
 * forwards since the last call, and resets.  flops / bytes are ALGORITHMIC (2*MAC of the true
 * convolution; activations + weights + outputs touched once). */
typedef struct {
  char name[32];
  int launches;      /* kernel launches aggregated */
  int forwards;      /* forwards aggregated */
  double ms;         /* summed device time */
  double flops;      /* summed algorithmic flops */
  double bytes;      /* summed algorithmic bytes */
} yb_prof_entry;
YB_API int yb_net_set_profiling(yb_net* net, int enable);
YB_API int yb_net_profile(yb_net* net, yb_prof_entry* out, int max_entries, int* num_entries);

/* One convolution layer of the engine as a standalone op (unit tests / per-layer parity at the
 * shapes of SURVEY.md App. A): y = [relu]( conv2d(x, w, stride, pad=k/2) + bias [+ residual] ).
 * x [B,Cin,H,H] and residual/out [B,Cout,Ho,Ho] are NCHW float32 on the DEVICE; w [Cout,Cin,k,k]
 * and bias [Cout] on the HOST.  k in {1,3}, stride in {1,2}, Cin % 64 == 0.  precision as in
 * yb_precision; use_tc = 1 selects the wgmma kernel (16-bit precisions only), 0 the CUDA-core
 * kernel.  Synchronous (allocates scratch internally). */
YB_API int yb_conv2d(const float* x, int batch, int cin, int h, const float* w, const float* bias, int cout, int k,
                     int stride, int relu, const float* residual, int precision, int use_tc, float* out);

/* End-to-end with HOST buffers: H2D(img) -> forward -> detect -> D2H(detections).
 * img_host [B,3,S,S]; outputs as in yb_detect (host).  The proto/coef needed for masks stay on
 * the device; yb_net_last_proto() exposes the proto of the last call. */
YB_API int yb_net_detect_host(yb_net* net, const float* img_host, int batch, const yb_detect_params* p,
                       int32_t* out_count, int32_t* out_class, int32_t* out_anchor,
                       float* out_score, float* out_box, float* out_coef);
YB_API const float* yb_net_last_proto(const yb_net* net);

/* Pipelined form of yb_net_detect_host for streams of batches: submit() enqueues
 * H2D(img) -> forward -> post-process -> D2H(records) on the net's own streams and returns at once;
 * collect() blocks until that submission's records are in the caller's buffers.  Up to two
 * submissions may be in flight, so the host->device copy of batch i+1 overlaps the compute of batch i.
 * img_host must stay valid (and should be pinned) until the matching collect() returns. */
YB_API int yb_net_submit_host(yb_net* net, const float* img_host, int batch, const yb_detect_params* p, int* ticket);
YB_API int yb_net_collect_host(yb_net* net, int ticket, int32_t* out_count, int32_t* out_class, int32_t* out_anchor,
                               float* out_score, float* out_box, float* out_coef);

/* ------------------------------------------------------------------------------------------
 * Training targets, losses and their gradients, batched -- replaces Yolact.compute_loss and the four loss functions
 * (modules/yolact.py:166-313) with utils/box_utils.py:57-114 match() / encode() and :147-168 crop().
 *   cls [B,A,C] RAW class logits, box [B,A,4], coef [B,A,K] (tanh applied), proto [B,P,P,K] (relu applied, NHWC),
 *   seg [B,Hs,Hs,ld_seg] segmentation logits, NHWC with row stride ld_seg >= C-1 (the reference's tensor is NCHW),
 *   anchors [A,4] (cx,cy,w,h), gt [total_gt,5] = (x1,y1,x2,y2 in [0,1], 0-based label) of all images back to back,
 *   gt_offset [B+1] int32 (image b owns rows gt_offset[b] .. gt_offset[b+1]), gt_masks [total_gt,S,S] float 0/1.
 * All pointers are DEVICE pointers except p (grad_scale: 4 DEVICE floats, NULL = ones).  losses[4] = (category, box, mask, semantic), weighted by
 * the *_alpha fields as the reference returns them.  The gradient outputs are optional (all NULL = losses only); they are the
 * derivatives of  sum_i grad_scale[i] * losses[i]  w.r.t. cls / box / coef (the tanh OUTPUT) / proto (the relu OUTPUT) / seg.
 * More than masks_to_train positives in an image: a uniformly random subset (counter-based hash of `seed`; the reference
 * draws torch.randperm, yolact.py:261-268).  dbg_* (optional): labels (>0 fg class+1, 0 bg, -1 neutral), matched gt index,
 * SSD offsets, mined-negative flags -- what match() / the OHEM step of the reference produce, for the parity tests.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  int batch, num_anchors, num_classes /* incl. background */, coef_dim, proto_size, seg_size, mask_size;
  float pos_iou_thr, neg_iou_thr;        /* cfg.pos_iou_thre / neg_iou_thre (config.py:103-104) */
  int neg_pos_ratio, masks_to_train;     /* 3 (yolact.py:205), cfg.masks_to_train (config.py:112) */
  float conf_alpha, bbox_alpha, mask_alpha, semantic_alpha;   /* config.py:106-109 */
} yb_loss_params;

YB_API size_t yb_losses_workspace_bytes(const yb_loss_params* p, int total_gt);
YB_API int yb_losses(const yb_loss_params* p, const float* cls, const float* box, const float* coef, const float* proto, const float* seg, int ld_seg,
                     const float* anchors, const float* gt, const int32_t* gt_offset, const float* gt_masks, int total_gt, int max_gt_per_image,
                     uint32_t seed, const float* grad_scale, float* losses, float* d_cls, float* d_box, float* d_coef, float* d_proto, float* d_seg,
                     int32_t* dbg_labels, int32_t* dbg_matched_idx, float* dbg_offsets, uint8_t* dbg_neg, void* workspace, size_t workspace_bytes,
                     void* stream);

/* ------------------------------------------------------------------------------------------
 * Training engine: Yolact.forward in training mode (modules/yolact.py:141-161) and its backward pass, ResNet-50/101 backbones.
 * Train-mode forward = wgmma convolutions on 16-bit activations + batch-statistics BatchNorm (running statistics updated in
 * place, momentum 0.1) + the loss kernels above; backward = dgrad convolutions and weight-gradient GEMMs on the same wgmma
 * kernel, BatchNorm / pooling / up-sampling backward on CUDA cores.  The fp32 master parameters stay where the caller keeps
 * them (torch nn.Parameters): yb_train_bind hands over DEVICE pointers to each parameter / buffer and to the fp32 buffer that
 * receives its gradient; nothing is copied, optimizers and DDP see one set of tensors.
 *   create -> param_info / bind (all) -> [forward -> backward]*
 * ---------------------------------------------------------------------------------------- */
typedef struct yb_train yb_train;
typedef struct {
  float pos_iou_thr, neg_iou_thr;
  int neg_pos_ratio, masks_to_train;
  float conf_alpha, bbox_alpha, mask_alpha, semantic_alpha;
  float bn_momentum, bn_eps;             /* torch defaults 0.1 / 1e-5 */
} yb_train_hparams;

/* precision: YB_PREC_BF16 (recommended: gradients need the exponent range) or YB_PREC_FP16 */
YB_API int yb_train_create(const yb_net_config* cfg, int batch, int precision, yb_train** out);
YB_API void yb_train_destroy(yb_train* t);
/* bindable tensors: kind 0 = parameter (data + gradient buffer), 1 = buffer (running_mean / running_var; no gradient) */
YB_API int yb_train_num_tensors(const yb_train* t);
YB_API int yb_train_tensor_info(const yb_train* t, int i, const char** name, int64_t* count, int* kind);
YB_API int yb_train_bind(yb_train* t, const char* name, float* data_device, float* grad_device);
YB_API int yb_train_set_anchors(yb_train* t, const float* anchors_host, int num_anchors);
/* img [B,3,S,S] float32 NCHW; gt / gt_offset / gt_masks as in yb_losses; losses[4] (device).  Asynchronous on `stream`. */
YB_API int yb_train_forward(yb_train* t, const float* img, const float* gt, const int32_t* gt_offset, const float* gt_masks, int total_gt,
                            int max_gt_per_image, const yb_train_hparams* hp, uint32_t seed, float* losses, void* stream);
/* gradients of sum_i loss_grad[i] * losses[i] (loss_grad: 4 DEVICE floats, NULL = ones) into the bound gradient buffers (overwritten) */
YB_API int yb_train_backward(yb_train* t, const float* loss_grad, void* stream);
/* debug / parity taps: copy a named activation (grad = 0) or its gradient (grad = 1) as NCHW float32 [B,C,H,H] (device) */
YB_API int yb_train_read(yb_train* t, const char* name, int grad, float* out, int64_t out_count, int* C, int* H, void* stream);
YB_API uint64_t yb_train_launches_per_step(const yb_train* t);

#ifdef __cplusplus
}
#endif
#endif /* YOLACT_B200_H_ */
