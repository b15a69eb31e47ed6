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

/* Class counts (num_classes, background included) every entry point accepts: 2 .. YB_MAX_CLASSES.  The bound comes from the
 * kernels that give each lane of a warp a fixed number of classes: C - 1 <= 128 foreground classes in the post-process, and
 * at most 5 logits per lane in the head softmax.  yb_net_create and yb_train_create refuse a larger count with
 * YB_ERR_UNSUPPORTED, yb_detect likewise, and yb_losses with YB_ERR_INVALID. */
#define YB_MAX_CLASSES 129

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

/* Batched mask assembly, bit-packed output (mask_f32 = 2 above) -- after_nms for the detect_batched record of B images of any
 * sizes, with no host sync on the detection counts.
 *   proto [B,P,P,K] (Yolact.forward's proto), coef [B,D,K], box [B,D,4], count [B] int32: detect_batched's record (DEVICE).
 *   img_hw [B,2] int32 (h, w) and mask_off [B+1] int64 are HOST tables: image b writes its masks [D,h_b,ceil(w_b/32)] words from
 *   out_mask + mask_off[b]; it owns D*h_b*ceil(w_b/32) words there, which must end at or before mask_off[b+1], and mask_off[B] <=
 *   mask_words.  Detections at or past count[b] write no mask words; their blocks exit at once.  out_box_px [B,D,4] int32 gets
 *   every row: trunc(box * max(h_b,w_b)) below count[b], zero at or past it.
 *   Image b's first count[b] masks and boxes equal yb_mask_assemble(mask_f32 = 2) on that image bit for bit.
 * Every size and offset is checked on the host before anything is launched (YB_ERR_INVALID); the geometry table is then copied
 * through library-owned page-locked staging (as yb_train_aug's), so the call queues without waiting for the stream.
 * workspace: B*D*P*P floats plus the table (yb_mask_assemble_batch_workspace_bytes) -- 487 MB at B = 64, D = 100, P = 138. */
YB_API size_t yb_mask_assemble_batch_workspace_bytes(int batch, int max_det, int proto_size);
YB_API int yb_mask_assemble_batch(const float* proto, const float* coef, const float* box, const int32_t* count, int batch, int max_det,
                                  int proto_size, int coef_dim, const int32_t* img_hw, const int64_t* mask_off, int64_t mask_words,
                                  int crop, void* workspace, size_t workspace_bytes, uint32_t* out_mask, int32_t* out_box_px,
                                  void* stream);

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
 * COCO's own mAP: pycocotools' COCOeval (default Params, iouType 'bbox' and 'segm') for the detections of eval.py's loop, which
 * --coco_api hands to pycocotools as JSON (eval.py:60-67,:78-98).  precision / recall equal COCOeval's float64 arrays bit for
 * bit (DESIGN.md, COCO mAP on the GPU):
 *   yb_cocoeval_match       per image: the detections the JSON would hold (class in range, (y2-y1)*(x2-x1) > 0), their rank
 *                           within (image, class) by descending score (ties: detection order), the first max_dets[2] of each
 *                           class kept; double IoUs against the image's gts of the same class (bbox: pycocotools' bbIou on xywh,
 *                           crowd gts divide by the detection's area; segm: popcounts of the packed masks); then COCOeval's greedy
 *                           matching for every slot (type, area range, IoU threshold).  Appends one record per kept detection
 *                           in a region of count[b] records at the running count plus the earlier images' counts (no host sync);
 *                           the unused tail of a region holds records of class -1.
 *   yb_cocoeval_accumulate  COCOeval.accumulate: a stable sort of the records by (class, descending score, image rank), then
 *                           per (type, IoU threshold, class, area range, maxDets) tp / fp counts in double, the running maximum
 *                           of precision from the right sampled at searchsorted(recall, rec_thr, 'left').  precision
 *                           [2][10][101][K][4][3] and recall [2][10][K][4][3] (type 0 = bbox, 1 = segm), -1 where npig = 0.
 * Limits: max_det <= 256; bits(num_classes) + bits(num_images - 1) <= 32 (the sort key), e.g. 2^25 images at 80 classes.
 * Inputs of yb_cocoeval_match (DEVICE pointers; batch B, max_det D, total_gt G):
 *   count [B], cls [B,D] (0-based class), score [B,D], box_px [B,D,4] int32 x1,y1,x2,y2; det_masks / det_mask_off [B+1] (int64
 *            words) / det_mask_words: at least count[b] packed masks of img_hw[b] = (h, w) per image, as yb_eval_match takes them
 *   img_rank [B] int32: the image's position in ascending image-id order, 0 .. num_images-1
 *   gt_cls [G] int32 (0-based class), gt_box [G,4] float64 x,y,w,h (the annotation's bbox), gt_area [G] float64 (its area),
 *            gt_crowd [G] int32; gt_offset [B+1]: image b owns gts gt_offset[b] .. gt_offset[b+1], every annotation of the image
 *            in file order, crowd included; gt_masks / gt_mask_off [B+1] / gt_mask_words: one packed mask per gt
 *   state [yb_cocoeval_state_bytes]: zeroed before the first batch.  Bytes 0-7: records appended so far (uint64); bytes 12-15:
 *            flags (bit 0: capacity exceeded, bit 1: an image's ranges lie outside the buffers or do not match its geometry,
 *            bit 2: an image rank outside 0 .. num_images-1; such images append records of class -1).
 * ---------------------------------------------------------------------------------------- */
#define YB_COCOEVAL_THR 10
#define YB_COCOEVAL_REC 101
#define YB_COCOEVAL_AREAS 4
#define YB_COCOEVAL_MAXDETS 3
typedef struct {
  int num_classes;                                /* K: len(catIds) */
  int num_images;                                 /* len(imgIds) */
  double iou_thr[YB_COCOEVAL_THR];                /* np.linspace(.5, .95, 10), made on the host */
  double rec_thr[YB_COCOEVAL_REC];                /* np.linspace(0, 1, 101) */
  double area_rng[YB_COCOEVAL_AREAS][2];          /* all / small / medium / large, both ends inclusive */
  int max_dets[YB_COCOEVAL_MAXDETS];              /* 1, 10, 100 (ascending, at most 256) */
} yb_cocoeval_params;

typedef struct {
  float score;
  int32_t cls;                     /* 0-based class; -1: no detection */
  int32_t img;                     /* image rank */
  int16_t det;                     /* detection index in the image */
  int16_t rank;                    /* rank within (image, class) */
  uint32_t bits[8];                /* [type * 4 + area]: bit t matched at iou_thr[t], bit 16 + t ignored */
} yb_cocoeval_record;

YB_API size_t yb_cocoeval_state_bytes(void);
YB_API size_t yb_cocoeval_match_workspace_bytes(int batch, int max_det, int64_t total_gt);
YB_API int yb_cocoeval_match(const yb_cocoeval_params* p, int batch, int max_det, const int32_t* count, const int32_t* cls,
                             const float* score, const int32_t* box_px, const uint32_t* det_masks, const int64_t* det_mask_off,
                             int64_t det_mask_words, const int32_t* img_hw, const int32_t* img_rank, const int32_t* gt_cls,
                             const double* gt_box, const double* gt_area, const int32_t* gt_crowd, const int32_t* gt_offset,
                             int64_t total_gt, const uint32_t* gt_masks, const int64_t* gt_mask_off, int64_t gt_mask_words,
                             yb_cocoeval_record* records, int64_t capacity, void* state, void* workspace, size_t workspace_bytes,
                             void* stream);
/* num_records: an upper bound of the records appended; npig [K][4] int64: non-ignored gts per (class, area range) over every image
 * of the annotation set */
YB_API size_t yb_cocoeval_accumulate_workspace_bytes(int64_t num_records);
YB_API int yb_cocoeval_accumulate(const yb_cocoeval_params* p, const yb_cocoeval_record* records, int64_t num_records, const void* state,
                                  const int64_t* npig, void* workspace, size_t workspace_bytes, double* precision, double* recall,
                                  void* stream);

/* ------------------------------------------------------------------------------------------
 * Pre-process -- replaces utils/augmentations.py:219-227 val_aug(img, val_size) (SURVEY.md 8(f) #1):
 * uint8 BGR HWC image [h,w,3] (device) -> float32 RGB CHW [3,S,S] (device): pad to square at the
 * top-left with the BGR mean, bilinear resize (OpenCV INTER_LINEAR coordinates), (x-mean)/std.
 * ---------------------------------------------------------------------------------------- */
YB_API int yb_val_aug(const uint8_t* img_bgr, int h, int w, int img_size, float* out, void* stream);

/* Batched form: src is one device buffer holding B uint8 BGR HWC images of any sizes; items is a HOST table, item i is the
 * image [h,w,3] at byte img_off of src and writes out[i] ([B,3,S,S] float32 RGB).  One launch; image i equals yb_val_aug on it
 * bit for bit.  Every offset and size is checked on the host before the launch (YB_ERR_INVALID); the table is then copied into
 * the workspace through the page-locked staging of yb_train_aug, so the call queues without waiting for the stream. */
typedef struct {
  int64_t img_off;           /* byte offset of the image in src */
  int32_t h, w;
} yb_val_aug_item;

YB_API size_t yb_val_aug_batch_workspace_bytes(int n_items);
YB_API int yb_val_aug_batch(const uint8_t* src, int64_t src_bytes, const yb_val_aug_item* items, int n_items, int img_size,
                            void* workspace, size_t workspace_bytes, float* out, void* stream);

/* ------------------------------------------------------------------------------------------
 * JPEG encoding -- cv2.imwrite / cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, quality]) of uint8 BGR images, byte for
 * byte: baseline, 4:2:0, ISLOW DCT, Annex K Huffman tables, JFIF header, no restart markers (oracle/jpeg_np.py).
 * src and items as yb_val_aug_batch (items is a HOST table, images of any sizes).  out_off is a HOST array of n + 1 byte offsets
 * into the device buffer out: file i is written at out[out_off[i] ..) and its length to out_len[i] (device); out_off[i+1] -
 * out_off[i] must be at least yb_jpeg_encode_bound(h, w).  No byte of out past out_off[i] + out_len[i] changes.  Every offset,
 * size and the quality (1 .. 100) are checked on the host before anything is launched (YB_ERR_INVALID); the tables then go
 * through the page-locked staging, so the call queues on the stream without waiting: five launches, no synchronisation.
 * ---------------------------------------------------------------------------------------- */
YB_API int64_t yb_jpeg_encode_bound(int h, int w);   /* worst-case file bytes of an h x w image (-1 outside 1 .. 65535) */
YB_API size_t yb_jpeg_encode_workspace_bytes(const yb_val_aug_item* items, int n);
YB_API int yb_jpeg_encode_batch(const uint8_t* src, int64_t src_bytes, const yb_val_aug_item* items, int n, int quality,
                                void* workspace, size_t workspace_bytes, uint8_t* out, const int64_t* out_off, int64_t* out_len,
                                void* stream);

/* ------------------------------------------------------------------------------------------
 * JPEG decoding -- cv2.imread(path) of a batch of JPEG files, pixel for pixel: libjpeg-turbo's ISLOW IDCT, fancy upsampling,
 * BGR output, then the EXIF orientation applied as OpenCV applies it (oracle/jpeg_decode_np.py).  Supported files: baseline or
 * extended-sequential Huffman, 8-bit, one scan holding every component, with or without restart intervals; grayscale, or YCbCr
 * with chroma 1x1 and luma 1x1, 2x1 or 2x2 (4:4:4, 4:2:2, 4:2:0).
 *
 * Host only: reads the markers of one file.  YB_OK with the output h, w (orientation applied) for a supported file,
 * YB_ERR_UNSUPPORTED for a valid JPEG outside the supported set, YB_ERR_INVALID for a malformed header. */
YB_API int yb_jpeg_header(const uint8_t* data, int64_t len, int32_t* h, int32_t* w);
/* File i is src[src_off[i] .. src_off[i+1]) (src_off a HOST array of n + 1 offsets), in both a HOST copy src_host (for the
 * headers) and a device copy src_dev (for the entropy-coded data).  Image i is written as uint8 BGR [h,w,3] at out + items[i].img_off
 * (items a HOST yb_val_aug_item table, the layout yb_val_aug_batch reads).  Headers, sizes against items and offsets are checked on
 * the host before anything is launched (YB_ERR_INVALID / YB_ERR_UNSUPPORTED, what yb_jpeg_header returns); the tables then go
 * through the page-locked staging, so the call queues without waiting: five launches, no synchronisation.
 * status (device int32 [n]): 0 for a clean decode; nonzero for corrupt entropy-coded data (an invalid code, a run past coefficient
 * 63, the wrong number of restart markers, too few blocks).  A corrupt stream never reads outside its file nor writes outside
 * its output slot; what the slot then holds is unspecified.  After the call the first n int32 of the workspace hold each file's
 * number of synchronisation rounds of the Huffman decode (0 for a file whose restart markers are wrong).
 * yb_jpeg_decode_workspace_bytes returns 0 if a header does not parse. */
YB_API size_t yb_jpeg_decode_workspace_bytes(const uint8_t* src_host, const int64_t* src_off, int n);
YB_API int yb_jpeg_decode_batch(const uint8_t* src_host, const uint8_t* src_dev, const int64_t* src_off, int n,
                                const yb_val_aug_item* items, uint8_t* out, int64_t out_bytes,
                                void* workspace, size_t workspace_bytes, int32_t* status, void* stream);

/* ------------------------------------------------------------------------------------------
 * Training augmentation -- the pixel work of utils/augmentations.py:230-252 train_aug for a batch, given the
 * plans drawn on the host by yolact_minimal_b200.utils.augmentations.train_aug_plan (every random draw of
 * train_aug depends only on shapes and boxes, so the host keeps them and the device only moves pixels).
 * Per output pixel, a composite gather:
 *   to_train_size pad/crop -> INTER_LINEAR resize square -> resize (OpenCV coordinates: x taps clamped with
 *   weight 0 outside, y rows clipped with the weights kept) -> pad to square (image fill norm_mean, mask 0)
 *   -> crop -> mirror -> photometric transform of the source pixel:
 *   brightness (+delta, clip 0..255), contrast (*alpha, clip), cv2 float BGR->HSV, S *= saturation (no clip),
 *   H += hue (wrapped once at > 360 / < 0), cv2 float HSV->BGR, clip 0..255; then (x-mean)/std, BGR->RGB.
 * Masks use float32 arithmetic, or (mask_u8 = 1, when the cropped image is already square and no pad made the
 * masks float) OpenCV's 11-bit fixed-point linear weights with its vectorised rounding
 * ((((h0>>4)*b0>>16) + ((h1>>4)*b1>>16) + 2) >> 2), which leaves them 0/1.
 *
 * src: one device buffer holding every image (uint8 BGR HWC [h,w,3]) and its masks (uint8 [num_masks,h,w]).
 * items / keep are HOST tables (copied into the workspace): item i writes out_img[i] ([B,3,S,S] float32 RGB) and
 * out_masks rows out_mask .. out_mask+num_keep-1 ([G,S,S] float32, G = sum of num_keep); row k is the source mask
 * keep[keep_begin + k].  Items are dense: out_mask and keep_begin both equal the sum of num_keep before the item.
 * Every offset, size and index is checked on the host before anything is launched (YB_ERR_INVALID).  The tables are
 * then copied through library-owned page-locked staging, so the call queues on the stream without waiting for earlier work;
 * the caller's tables may be freed when it returns.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  int64_t img_off;           /* byte offset of the image in src */
  int64_t mask_off;          /* byte offset of the masks in src */
  int32_t h, w, num_masks;
  int32_t brightness_on;     /* 0/1 */
  float brightness_delta;    /* float32, added when brightness_on */
  int32_t contrast_on;       /* 0/1 */
  float contrast_alpha;      /* float32, multiplied when contrast_on */
  float saturation_scale;
  float hue_delta;
  int32_t mirror;            /* 0/1: x -> w-1-x before the crop */
  int32_t crop_x, crop_y, crop_w, crop_h; /* crop rectangle in the (mirrored) image; (0,0,w,h) when not cropped */
  int32_t square;            /* max(crop_w, crop_h) */
  int32_t pad_x, pad_y;      /* offset of the crop in the square */
  int32_t resize;            /* side after the multi-scale resize */
  int32_t train_x, train_y;  /* to_train_size: pad offset when resize < img_size, crop offset when resize > img_size, else 0 */
  int32_t mask_u8;           /* 0 float32 mask arithmetic, 1 OpenCV uint8 fixed point */
  int32_t out_mask, keep_begin, num_keep;
} yb_train_aug_item;

YB_API size_t yb_train_aug_workspace_bytes(int n_items, int64_t n_keep);
YB_API int yb_train_aug(const uint8_t* src, int64_t src_bytes, const yb_train_aug_item* items, int n_items, const int32_t* keep,
                        int img_size, void* workspace, size_t workspace_bytes, float* out_img, float* out_masks, void* stream);

/* ------------------------------------------------------------------------------------------
 * Drawing -- the pixel work of utils/output_utils.py:308-369 (draw_img); the box, label and fps drawing stays on the host.
 *   semantic = (sum_i m_i * (ids_i + 1)) mod num_colors     floor modulo (numpy %); num_colors = cfg.num_classes - 1
 *   yb_draw_masks   out = rint(0.4f * palette[semantic] + 0.6f * img) per channel -- cv2.addWeighted(COLORS[semantic], 0.4,
 *                   img, 0.6, 0) on uint8, every pixel (the background blends with palette[0]); one launch
 *   yb_draw_cutout  cfg.cutout: out_total = semantic != 0 ? img : 255 ([h,w,3]); crop i = (m_i != 0 ? img : 255) over rows
 *                   crop_yyxx[i] = (y1, y2, x1, x2) -> cols [x1, x2), written [y2-y1, x2-x1, 3] at out_crops + crop_off[i]
 *                   (int64 byte offsets [n+1]).  A crop outside the image, or whose range crop_off[i] .. crop_off[i+1] does not
 *                   hold exactly its 3 * area bytes, is skipped (nothing is written for it).
 * img_bgr / out_* uint8 [h,w,3] (HWC, any channel order: channel c of the palette applies to channel c of the image);
 * masks [n,h,w] with values {0,1} in the layouts of yb_mask_assemble (mask_fmt 0 uint8, 1 float32 -- 16-byte aligned, 2
 * bit-packed words [n,h,ceil(w/32)]); ids int32 [n]; palette uint8 [num_colors,3].  n <= 4096, 1 <= num_colors <= 1024.
 * All pointers are DEVICE pointers; asynchronous on stream.  out_bgr may alias img_bgr.
 * ---------------------------------------------------------------------------------------- */
YB_API int yb_draw_masks(const uint8_t* img_bgr, int h, int w, const void* masks, int mask_fmt, int n, const int32_t* ids,
                         const uint8_t* palette, int num_colors, uint8_t* out_bgr, void* stream);
YB_API int yb_draw_cutout(const uint8_t* img_bgr, int h, int w, const void* masks, int mask_fmt, int n, const int32_t* ids,
                          int num_colors, const int32_t* crop_yyxx, const int64_t* crop_off, uint8_t* out_total,
                          uint8_t* out_crops, void* stream);

/* Batched overlay: yb_draw_masks for B images of any sizes in one launch, with no host sync on the detection counts.
 *   src / items: the raw images back to back and their HOST yb_val_aug_item table (the buffer yb_val_aug_batch reads); out
 *   (src_bytes bytes, same layout) must not overlap src.  masks: bit-packed, image b's [max_det, h_b, ceil(w_b/32)] words from
 *   masks + mask_off[b] (HOST int64 [B+1]; they must end at or before mask_off[b+1], and mask_off[B] <= mask_words):
 *   yb_mask_assemble_batch's buffer.  ids int32 [B, max_det]; count int32 [B] (DEVICE).
 *   Image b blends its first min(count[b], max_det) masks exactly as yb_draw_masks does; an image with count[b] <= 0 is copied
 *   unchanged (draw_img returns img_origin when nothing is left).
 * Every size and offset is checked on the host before the launch (YB_ERR_INVALID); the geometry table then goes through the
 * page-locked staging of yb_mask_assemble_batch, so the call queues without waiting for the stream.
 * workspace: yb_draw_masks_batch_workspace_bytes(B). */
YB_API size_t yb_draw_masks_batch_workspace_bytes(int batch);
YB_API int yb_draw_masks_batch(const uint8_t* src, int64_t src_bytes, const yb_val_aug_item* items, int batch, const uint32_t* masks,
                               const int64_t* mask_off, int64_t mask_words, int max_det, const int32_t* ids, const int32_t* count,
                               const uint8_t* palette, int num_colors, void* workspace, size_t workspace_bytes, uint8_t* out,
                               void* stream);

/* cfg.save_lincomb: utils/output_utils.py:276-305 draw_lincomb for detection 0 of each of B images, one launch.
 *   proto float32 [B,P,P,K], coef float32 [B,max_det,K], count int32 [B] (DEVICE; NULL = every image): an image with
 *   count <= 0 is not written.  lut uint8 [256,3] (cv2.COLORMAP_WINTER); out uint8 [B, 4P, 8P, 3].  K must be 32
 *   (the 4 x 8 grid; anything else is YB_ERR_UNSUPPORTED).
 *   Cell (r, c) shows channel ch = order[8r + c], order = the 32 coefficients by |coef| descending, ties to the lower channel
 *   (NaN last): x = fp32(fp32(proto[y,x,ch] / max_ch) * coef[ch]) with max_ch the channel's maximum over its P x P plane (NaN if
 *   it holds one), u = ((double)x + 1) * 127.5, byte = low byte of the int32 truncation of u (x86-64's cast: NaN and values
 *   outside int32 give 0), pixel = lut[byte].  The reference's tie order is numpy's unstable argsort; this one is stable. */
YB_API int yb_draw_lincomb(const float* proto, const float* coef, const int32_t* count, int batch, int max_det, int proto_size,
                           int coef_dim, const uint8_t* lut, uint8_t* out, void* stream);

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

/* Debug: the finalized forward op by op (tests).  The program is the list of ops yb_net_forward runs, after the fusion of
 * bottleneck pairs; ops read and write activations by id.  yb_net_forward(...) == yb_net_forward_range(..., 0, num_ops, ...). */
typedef enum {
  YB_OP_STEM = 0, YB_OP_POOL, YB_OP_SPLIT, YB_OP_CONV, YB_OP_UPADD, YB_OP_UP2X, YB_OP_HEADFIN, YB_OP_PATCH_EMBED, YB_OP_LN,
  YB_OP_ATTN, YB_OP_MERGE_LN, YB_OP_BNECK
} yb_op_kind;

typedef struct {
  int kind;                            /* yb_op_kind */
  int in, out, res, aux, in2, out2;    /* activation ids, -1 = none.  STEM: aux = the space-to-depth image; UPADD: out is updated in
                                          place; BNECK: out = x', out2 = t1 of the next block, in2 = the folded downsample's input */
  int stride, relu, heads, shift, level;   /* relu: 0 none, 1 ReLU, 2 exact GELU; level: HEADFIN's pyramid level */
  int convd;                           /* BNECK: 1 = the block's 1x1 downsample convolution is folded into the first GEMM */
  int out_mode;                        /* CONV: 0 haloed activation, 1 dense fp32 rows */
  int ext_proto;                       /* CONV: 1 = writes the proto output of the forward (out = -1) */
  int k, cin, cout, cout_pad;          /* CONV / BNECK: the (first) convolution */
  int anchor_offset;                   /* HEADFIN: first anchor of the level */
  /* state-dict names ("" = none; valid until yb_net_destroy): conv weight / bias / BatchNorm prefix (the head's convolution, which
     concatenates conf | bbox | coef, has none), BNECK's second convolution and folded downsample, Swin parameter vectors
     (LN / MERGE_LN: weight, bias; ATTN: qkv bias, relative-position table) */
  const char* w0; const char* b0; const char* bn0;
  const char* w1; const char* bn1;
  const char* wd; const char* bnd;
  const char* p0; const char* p1;
} yb_op_info;

typedef struct {
  int C, H;                /* channels, valid side */
  int planes;              /* parity planes (stride-2 convolution inputs), else 1 */
  int dtype;               /* yb_precision code of the stored elements */
  int dense;               /* 1: dense fp32 rows [B*H*H][C] without halo */
  int pad_rows;            /* rows allocated behind the max_batch images (the stem's space-to-depth image) */
  int64_t plane_rows;      /* rows between parity planes: max_batch * (H+2)^2 */
} yb_act_info;

YB_API int yb_net_num_ops(const yb_net* net);
YB_API int yb_net_op_info(const yb_net* net, int op, yb_op_info* out);
YB_API int yb_net_num_acts(const yb_net* net);
YB_API int yb_net_act_info(const yb_net* net, int act, yb_act_info* out);
/* Copy activation `act` of the first `batch` images exactly as stored into dst (device), `bytes` = its exact size:
 *   haloed    [planes][batch][(H+2)^2][C] in the act dtype (planes taken at their plane_rows stride), followed by the pad_rows
 *             rows behind image batch-1 ([pad_rows][C]) when pad_rows > 0
 *   dense     [batch*H*H][C] fp32 */
YB_API int yb_net_read_act_raw(yb_net* net, int act, int batch, void* dst, size_t bytes, void* stream);
/* The packed GEMM operands of op `op` (device copies into w / b; NULL = sizes only):
 *   which = 0: CONV: [rows][cols] = [Cout rounded up to 64][k*k*Cin_pad] weights (BN folded, act dtype) and [rows] fp32 biases;
 *              BNECK: conv3, or [W3 | Wd] and b3 + bd with a folded downsample; STEM: the 16-bit [64][256] GEMM weights
 *   which = 1: BNECK: the next block's conv1 */
YB_API int yb_net_read_op_weights(yb_net* net, int op, int which, void* w, size_t w_bytes, float* b, size_t b_bytes, int* rows, int* cols,
                                  void* stream);
/* ops [first, last) of yb_net_forward, exactly as it runs them (arguments as there) */
YB_API int yb_net_forward_range(yb_net* net, const float* img, int batch, int first, int last, float* cls, float* box, float* coef,
                                float* proto, void* stream);

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
 * Training engine: Yolact.forward in training mode (modules/yolact.py:141-161) and its backward pass, ResNet-50/101 and Swin-T
 * (depth 0: no BatchNorm buffers; stochastic depth drawn on the device from `seed`) backbones.
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
/* debug / parity taps: copy a named activation (grad = 0) or its gradient (grad = 1) as NCHW float32 [B,C,H,H] (device).
 * Swin-T names: "patch_embed"; per block P = "backbone.layers.<s>.blocks.<b>": P".norm1", P".attn.qkv" (q | k | v, 3C channels),
 * P".attn" (attention output), P".attn.proj", P".x1" (after the attention residual), P".norm2", P".mlp.fc1" (before GELU),
 * P".mlp.gelu", P".mlp.fc2", P".out"; per merge D = "backbone.layers.<s>.downsample": D".merge" (gathered 4C tokens), D".norm",
 * D".reduction"; "c3" / "c4" / "c5" (backbone.norm1..3).  "out.drop_path": the step's stochastic-depth masks [B,12,2] (block,
 * attention | MLP), C = 2, H = 12, no gradient; the "out.*" network outputs likewise. */
YB_API int yb_train_read(yb_train* t, const char* name, int grad, float* out, int64_t out_count, int* C, int* H, void* stream);
YB_API uint64_t yb_train_launches_per_step(const yb_train* t);

/* ------------------------------------------------------------------------------------------
 * Optimizer step: torch's foreach SGD (momentum, L2 weight decay, dampening 0) and AdamW (decoupled weight decay) on CUDA,
 * bit for bit, over every parameter in one launch.  The parameters stay where the caller keeps them (params_device[i],
 * counts[i] fp32 elements); their gradient is ONE flat fp32 buffer, the parameters concatenated in the order given here (the
 * order of a yb_train program's kind-0 tensors, so yb_train_bind's gradient buffer can be passed as is).  The optimizer owns
 * its state (SGD: momentum buffer; AdamW: exp_avg, exp_avg_sq; zero at creation) and does not belong to a yb_train: several
 * programs (batch sizes) bound to the same parameters step the same state.
 *   create -> [step]* -> destroy
 * yb_optim_step: p <- update(p, grad_scale * grad_flat) with learning rate `lr`; the per-step scalars (bias corrections) are
 * computed on the host in double from the call count, as torch computes them.  Asynchronous on `stream`; touches nothing
 * outside the listed parameter ranges.  Must run on the device the optimizer was created on.
 * ---------------------------------------------------------------------------------------- */
typedef struct yb_optim yb_optim;
typedef enum { YB_OPTIM_SGD = 0, YB_OPTIM_ADAMW = 1 } yb_optim_kind;
typedef struct {
  int kind;                              /* yb_optim_kind */
  double momentum, dampening;            /* SGD: momentum > 0, dampening 0 */
  double weight_decay;                   /* SGD: added to the gradient; AdamW: decoupled (p *= 1 - lr * weight_decay) */
  double beta1, beta2, eps;              /* AdamW: 0.5 < beta1 < 1, 0 <= beta2 < 1 */
} yb_optim_params;

YB_API int yb_optim_create(const yb_optim_params* p, int n, float* const* params_device, const int64_t* counts, yb_optim** out);
YB_API int yb_optim_step(yb_optim* o, const float* grad_flat, double lr, float grad_scale, void* stream);
/* debug / parity tap: state `which` (0: SGD momentum buffer | AdamW exp_avg, 1: AdamW exp_avg_sq) in the gradient's layout,
 * out_count = yb_optim_num_elements (device; asynchronous on `stream`) */
YB_API int yb_optim_read_state(const yb_optim* o, int which, float* out, int64_t out_count, void* stream);
/* elements of the flat gradient (sum of counts) */
YB_API int64_t yb_optim_num_elements(const yb_optim* o);
YB_API void yb_optim_destroy(yb_optim* o);

#ifdef __cplusplus
}
#endif
#endif /* YOLACT_B200_H_ */
