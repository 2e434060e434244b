/*
 * ryolo.h -- C-ABI of the H100-native rotate-yolov3 hot path (libryolo.so).
 *
 * Every entry point is `extern "C"`, takes plain pointers / sizes / a CUDA stream handle
 * (passed as void* so that this header needs no CUDA include), allocates nothing behind the
 * caller's back (scratch comes from a caller-owned workspace whose size is queried first),
 * never throws, and returns an int status: 0 = ok, <0 = RYOLO_E_* (see ryolo_last_error()).
 * All data pointers are DEVICE pointers unless the parameter name ends in `_host`.
 * There is NO CPU fallback: without a CUDA device every compute call returns RYOLO_E_CUDA.
 *
 * Reference interfaces replaced (paths relative to the reference repo, ming71/rotate-yolov3):
 *   ryolo_rnms*            <- r_nms(dets, thr)          utils/nms/src/rotate_polygon_nms.cpp:7-16
 *                             nms_cuda()                utils/nms/src/rotate_polygon_nms_kernel.cu:323-384
 *                             rotate_nms_kernel         utils/nms/src/rotate_polygon_nms_kernel.cu:262-308
 *   ryolo_riou_*           <- skew_bbox_iou(box1, box2, GIoU)   utils/utils.py:290-320
 *                             skewiou / get_rotated_coors        utils/utils.py:663-699, 702-725
 *   ryolo_nms_filter       <- non_max_suppression() candidate filter  utils/nms/nms.py:34-40,55
 *   ryolo_conv_*           <- Conv2d -> BatchNorm2d -> PReLU blocks built by create_modules
 *                             model/models.py:49-66; folded BN per utils/torch_utils.py:45-69
 *   ryolo_yolo_decode      <- YOLOLayer.forward eval branch   model/models.py:183-227,
 *                             create_grids                     model/model_utils.py:16-35
 */
#ifndef RYOLO_H_
#define RYOLO_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RYOLO_OK 0
#define RYOLO_E_ARG (-1)       /* bad argument (null pointer, negative size, unknown mode) */
#define RYOLO_E_WORKSPACE (-2) /* workspace too small / misaligned                          */
#define RYOLO_E_CUDA (-3)      /* CUDA runtime error (text in ryolo_last_error)             */
#define RYOLO_E_UNSUPPORTED (-4)

/* ABI version of this header; bumped on any signature change. */
int ryolo_abi_version(void);
/* Thread-local text of the last failure on the calling thread ("" if none). */
const char* ryolo_last_error(void);
/* Number of this library's kernel launches issued by the calling process so far
 * (bench.py's `gpu_launches` evidence). */
uint64_t ryolo_launch_count(void);
/* Keep n SMs free of this library's persistent GEMM kernels (conv fwd / dgrad / wgrad grids = SM count - n) from now on:
 * a data-parallel training step reserves a few SMs during backward so that the concurrent NCCL all-reduce kernels are
 * resident next to them instead of forcing a second wave (process-wide setting, 0 <= n <= 64; 0 = use every SM). */
int ryolo_set_reserved_sms(int n);

/* ------------------------------------------------------------------------------------------ *
 * Rotated NMS  (reference: r_nms / nms_cuda, rotate_polygon_nms_kernel.cu:323-384)
 *
 * dets     [n,6] fp32 (cx, cy, w, h, theta_rad, score), row-major, device.
 * thr      suppress j iff IoU(i,j) > thr (strict), i = higher score; NaN IoU never suppresses.
 * keep_out [n] int64, device: receives the ORIGINAL indices of the kept boxes, ASCENDING
 *          (reference :380-383); only the first *num_keep entries are defined.
 * num_keep device int32[1].
 * The IoU arithmetic replicates the reference device code operation-for-operation, including
 * the FMA contractions nvcc's default -fmad=true applies to it (DESIGN.md "pinned arithmetic"),
 * so the kept index list is bit-identical to the reference kernel's on the same inputs when the
 * scores are tie-free (the reference's torch sort is unstable; ours is a stable descending sort).
 * The mask is evaluated lazily in row chunks of 1024 boxes, alternating with the greedy scan:
 * rows and columns already suppressed by earlier chunks are skipped -- their mask bits can never
 * influence the scan, so the kept list is unchanged while dense candidate sets cost far less.
 * Asynchronous on `stream`; no host synchronisation inside.
 * ------------------------------------------------------------------------------------------ */
size_t ryolo_rnms_workspace_bytes(int n);
int ryolo_rnms(const float* dets, int n, float thr, int64_t* keep_out, int32_t* num_keep,
               void* workspace, size_t workspace_bytes, void* stream);

/* Same result as ryolo_rnms, but computes EVERY upper-triangle mask word in one launch like the
 * reference kernel (no skipping of already-suppressed rows/columns).  Slower; exists so that the
 * parity tests can compare the whole mask with the reference's. */
int ryolo_rnms_full_mask(const float* dets, int n, float thr, int64_t* keep_out, int32_t* num_keep,
                         void* workspace, size_t workspace_bytes, void* stream);

/* Batched ("segmented") form: `segments` independent NMS problems -- one per (image, class) -- in ONE set of launches
 * (reference: the per-image / per-class Python loop of non_max_suppression, utils/nms/nms.py:28-69, calling r_nms once
 * per class).  Segment s owns rows [s*cap, s*cap + n_dev[s]) of dets [segments*cap, 6]; its counts come from DEVICE
 * memory (ryolo_detect_select), so nothing synchronises with the host.  At most `limit` boxes per segment -- the
 * best-scored, ties by row index -- enter the NMS.  keep_out [segments, cap] int64: kept row indices WITHIN the segment,
 * ascending; num_keep [segments] int32.  Same kernels and same pinned arithmetic as ryolo_rnms (which is the
 * segments = 1, host-count case): per segment the kept list is bit-identical to r_nms on that segment's boxes. */
size_t ryolo_rnms_batched_workspace_bytes(int segments, int cap);
int ryolo_rnms_batched(const float* dets, int segments, int cap, const int32_t* n_dev, int limit, float thr,
                       int64_t* keep_out, int32_t* num_keep, void* workspace, size_t workspace_bytes,
                       void* stream);

/* Batched candidate selection in front of it (reference: utils/nms/nms.py:34-40 per image; detect.py:204-213).
 * io [batch, p, 6+nc] fp32 decoded predictions (NOT modified).  Per image: of the rows passing the reference's filter
 * (conf = obj * max class conf > conf_thres, w and h > min_wh, all values finite), exactly the `limit` with the largest
 * conf -- ties resolved by lowest row index -- are written IN INPUT ORDER to dets_out [batch, cap, 6] =
 * (x, y, w, h, theta, conf); n_out [batch] int32 = min(limit, rows passing).  cap >= limit is the row stride of
 * dets_out.  conf_thres must be >= 0 (RYOLO_E_ARG otherwise, NaN included). */
size_t ryolo_detect_select_workspace_bytes(int batch, int p);
int ryolo_detect_select(const float* io, int batch, int p, int nc, float conf_thres, float min_wh, int limit,
                        float* dets_out, int cap, int32_t* n_out, void* workspace, size_t workspace_bytes,
                        void* stream);

/* Class-aware forms, for configs with any number of classes (reference: the per-class loop of non_max_suppression,
 * utils/nms/nms.py:47-56).
 * ryolo_detect_select_classes: the same selection as ryolo_detect_select, written as 8 columns dets_out
 * [batch, cap, 8] = (x, y, w, h, theta, conf, class_conf, class): class_conf, class = max / first argmax of the class
 * scores.  Workspace: ryolo_detect_select_workspace_bytes.  nc must be <= 2^24.
 * ryolo_rnms_batched_classes: one NMS per class within each segment, in one set of launches.  dets8 [segments, cap, 8]
 * with the score in column 5 and the class id in column 7; all n_dev[s] rows of segment s enter.  Each segment is sorted
 * by (class asc, score desc, row asc) and the suppression mask only holds same-class pairs, so its memory is that of
 * ryolo_rnms_batched at the same cap, whatever the number of classes.  keep_out / num_keep as ryolo_rnms_batched:
 * kept row indices within the segment, ascending; per class, the kept list is bit-identical to ryolo_rnms on that
 * class's rows.  Class ids must be integers in [0, 2^24) and scores > 0: a row that breaks this (checked on the
 * device) is never suppressed and suppresses nothing. */
int ryolo_detect_select_classes(const float* io, int batch, int p, int nc, float conf_thres, float min_wh, int limit,
                                float* dets_out, int cap, int32_t* n_out, void* workspace, size_t workspace_bytes,
                                void* stream);
size_t ryolo_rnms_batched_classes_workspace_bytes(int segments, int cap);
int ryolo_rnms_batched_classes(const float* dets8, int segments, int cap, const int32_t* n_dev, float thr,
                               int64_t* keep_out, int32_t* num_keep, void* workspace, size_t workspace_bytes,
                               void* stream);

/* Cross-scale merge of multi-scale detection (reference: multi_detect, detect.py:81-101): the kept rows of `scales`
 * results of ryolo_detect_select_classes + ryolo_rnms_batched_classes, mapped back to original-image pixels and
 * concatenated per image.  dets_host / keep_host / num_keep_host: host arrays of `scales` device pointers, result s
 * being dets [batch, cap, 8], keep [batch, cap] int64 and num_keep [batch] int32.  table [scales, batch, 3] fp32 =
 * (padx, pady, gain) of each scale and image (the reference's scale_coords).  out [batch, scales * cap, 8]: image b's
 * rows are result 0's kept rows dets[b, keep[b, i]] for i < num_keep[b], then result 1's, ... (the offsets are prefix
 * sums of num_keep on the device), each with x = rint((x - padx) / gain), y = rint((y - pady) / gain),
 * w = rint(w / gain), h = rint(h / gain) in fp32 (rint: half to even) and theta, conf, class_conf, class copied; the
 * rest of the image's rows are zero (conf 0: no conf_thres >= 0 selects them).  1 <= scales <= RYOLO_MERGE_MAX_SCALES,
 * batch <= 65535.  Allocates nothing; capturable in a CUDA graph. */
#define RYOLO_MERGE_MAX_SCALES 16
int ryolo_merge_scales(const float* const* dets_host, const int64_t* const* keep_host,
                       const int32_t* const* num_keep_host, int scales, int batch, int cap, const float* table,
                       float* out, void* stream);

/* Introspection of the last ryolo_rnms_full_mask call that used `workspace` (valid until the workspace is
 * reused): device pointers to the score-sorted boxes [n,6], the sort permutation order[n]
 * (int32, sorted position -> original index) and the suppression mask [n, ceil(n/64)] uint64 in the
 * reference's layout (only words with column-block >= row-block are defined, as in the
 * reference host scan :371-374).  Used by the parity tests to compare masks bit-for-bit. */
int ryolo_rnms_debug_views(void* workspace, int n, const float** sorted_boxes,
                           const int32_t** order, const unsigned long long** mask);

/* ------------------------------------------------------------------------------------------ *
 * Rotated IoU  (reference: skew_bbox_iou, utils/utils.py:290-320)
 *
 * Boxes are rows of `stride` floats (stride >= 5) whose first five are (cx, cy, w, h, theta_rad);
 * corners per get_rotated_coors (utils/utils.py:702-725).  mode: 0 = 'iou'
 * (inter / (A1 + A2 - inter)), 1 = 'giou' as the reference defines it (inter / area of the
 * axis-aligned envelope of the 8 corners, utils/utils.py:682-685).  Zero-area boxes and a zero
 * denominator give 0 (utils/utils.py:672-673, 693-694).  fp32 in/out; geometry is an fp32
 * convex clip in box1's local frame (tolerance vs the float64 oracle: 1e-4 rel + 1e-6 abs).
 * ------------------------------------------------------------------------------------------ */
#define RYOLO_IOU_MODE_IOU 0
#define RYOLO_IOU_MODE_GIOU 1
/* out[i] = iou(a_i, b_i), i < n  (the reference's N-vs-N form) */
int ryolo_riou_paired(const float* a, const float* b, int n, int stride_a, int stride_b, int mode,
                      float* out, void* stream);
/* out[i*m + j] = iou(a_i, b_j)  (the reference's 1-vs-N form applied to every row of a) */
int ryolo_riou_pairwise(const float* a, int n, int stride_a, const float* b, int m, int stride_b,
                        int mode, float* out, void* stream);

/* Rotated IoU as a differentiable op (SURVEY.md 8f item 4: the README's "riou loss", which model/loss.py does not
 * implement): iou_out[i] = IoU(a_i, b_i) (mode 'iou' semantics as above) and, given grad_out[i] = dL/d iou_i (NULL = 1),
 * the analytic gradients grad_a / grad_b [n, 5] w.r.t. (cx, cy, w, h, theta) of each box (boundary-velocity formula:
 * d area(a ∩ b) = integral over the part of the moving box's boundary inside the other box of its normal velocity;
 * riou_grad.cu).  Any of iou_out / grad_a / grad_b may be NULL. */
int ryolo_riou_paired_grad(const float* a, const float* b, int n, int stride_a, int stride_b,
                           const float* grad_out, float* iou_out, float* grad_a, float* grad_b, void* stream);

/* Greedy prediction <-> ground-truth assignment of the mAP evaluation (reference test.py:134-151) on the device.
 * iou [p, t] (row stride iou_stride) = ryolo_riou_pairwise of the image's confidence-sorted predictions against its
 * targets; pcls: class of prediction i at pcls[i * pcls_stride]; tcls [t].  In order, a prediction is correct when the
 * best-IoU target OF ITS CLASS (first maximum) has IoU > iou_thres and was not claimed before; the walk stops once every
 * target is claimed.  correct [p] uint8; claimed_scratch [t] uint8. */
int ryolo_match_detections(const float* iou, int p, int t, int iou_stride, const float* pcls, int pcls_stride,
                           const float* tcls, float iou_thres, unsigned char* claimed_scratch,
                           unsigned char* correct, void* stream);

/* The same assignment for every image of a batch, straight from ryolo_detect_select_classes + ryolo_rnms_batched_classes
 * and with nothing read back to the host (reference test.py:80-151 after non_max_suppression).
 * dets8 [batch, cap, 8], keep [batch, cap], num_keep [batch]: their output (image b keeps rows keep[b, :num_keep[b]]).
 * targets [nt, 7] = (image, class, x, y, w, h, theta), x / w normalised by width and y / h by height (letterbox_labels);
 * image b's targets are the rows with image == b, in row order (rows of other image values belong to no image), scaled to
 * pixels as test.py:131-133 does.  Each image's kept rows are ordered by confidence descending, class ascending, then row
 * (a stable segmented sort: the order of nms.detections_per_image), its IoU matrix against its targets is computed with
 * ryolo_riou_pairwise's arithmetic, bit for bit, and walked as ryolo_match_detections does.
 * Output: image b's rows go to correct / conf / pcls [*count + sum of the earlier images' num_keep, ...) in that order
 * (correct uint8, conf = column 5, pcls = column 7), and *count (device int32) is advanced by the batch's kept rows.
 * class_hist (NULL = none) [nc + 1] int32: += the number of targets (of images 0..batch-1) per class, the last entry
 * counting classes that are not integers in [0, nc).  iou_scratch [cap * nt] fp32: image b's matrix, row stride t_b (its
 * target count), starts at cap * (targets of the images before b).  batch <= 4096; class ids < 2^24.
 * workspace == NULL: writes the workspace size to *workspace_bytes and returns (needs the device, which sizes the sort). */
int ryolo_match_batched(const float* dets8, const int64_t* keep, const int32_t* num_keep, int batch, int cap,
                        const float* targets, int nt, int height, int width, float iou_thres, unsigned char* correct,
                        float* conf, float* pcls, int32_t* count, int32_t* class_hist, int nc, float* iou_scratch,
                        void* workspace, size_t* workspace_bytes, void* stream);

/* ap_per_class (reference utils/utils.py:200-286) over the first *n_rows of n_cap rows (correct, conf, pcls as
 * ryolo_match_batched writes them), with n_gt [nc] targets per class.  out [nc, 4] float64 = (p, r, ap, f1) of each class;
 * a class with n_gt == 0 is not one of the reference's classes and gets zeros.  Rows are ordered by a stable sort on
 * confidence, descending: ties keep their row order (the reference's np.argsort(-conf) leaves it unspecified).  p, r and
 * f1 are the reference's float64 values; AP sums its terms in row order (the reference's np.sum is pairwise).  No float
 * atomics: the results repeat bit for bit.  workspace == NULL: writes the size to *workspace_bytes and returns. */
int ryolo_ap_per_class(const unsigned char* correct, const float* conf, const float* pcls, const int32_t* n_rows,
                       int n_cap, const int32_t* n_gt, int nc, double* out, void* workspace, size_t* workspace_bytes,
                       void* stream);

/* ------------------------------------------------------------------------------------------ *
 * non_max_suppression candidate filter (reference: utils/nms/nms.py:34-40, 55)
 *
 * pred [p, 6+nc] fp32 (x,y,w,h,theta,obj, cls...), one image.  Exactly like the reference:
 * class_conf/class_pred = max/argmax over the class columns (first max on ties), pred[:,5] *=
 * class_conf IN PLACE (nms.py:35), keep rows with conf > conf_thres, w > min_wh, h > min_wh and
 * all 6+nc values finite.  Survivors are written in input order to out [*, 8] =
 * (x,y,w,h,theta,conf,class_conf,class) and counted in num_out (device int32[1]).
 * Stable (order-preserving) compaction; capacity = max rows `out` can hold (extra rows dropped,
 * num_out still reports the true count so that the caller can detect overflow).
 * ------------------------------------------------------------------------------------------ */
size_t ryolo_nms_filter_workspace_bytes(int p);
int ryolo_nms_filter(float* pred, int p, int nc, float conf_thres, float min_wh, float* out,
                     int capacity, int32_t* num_out, void* workspace, size_t workspace_bytes,
                     void* stream);

/* ------------------------------------------------------------------------------------------ *
 * YOLO head decode (reference: YOLOLayer.forward eval branch, model/models.py:198-227)
 *
 * p        [bs, na*(nc+6), ny, nx] fp32 NCHW raw head output (the conv's natural layout).
 * anchors  [na, 3] fp32 (w_px, h_px, theta): anchor_vec = (w/stride, h/stride, theta)
 *          (model/model_utils.py:30-32).
 * io_out   [bs, io_rows_total, nc+6] fp32; this layer writes rows [row_offset, row_offset+na*ny*nx)
 *          of every image, in the reference's (a, y, x) order, so the three layers concatenate
 *          by row_offset exactly like torch.cat(io, 1) (model/models.py:298).
 * p_out    optional [bs, na, ny, nx, nc+6] fp32 permuted raw copy (the second tensor the
 *          reference returns); may be NULL.
 * arc_default != 0 -> sigmoid on obj and class columns ('default' arcs); nc == 1 forces the
 * class column to 1 (models.py:220-221).
 * ------------------------------------------------------------------------------------------ */
int ryolo_yolo_decode(const float* p, int bs, int na, int nc, int ny, int nx, const float* anchors,
                      float stride, float context_factor, int arc_default, float* io_out,
                      int io_rows_total, int row_offset, float* p_out, void* stream);

/* ------------------------------------------------------------------------------------------ *
 * Conv2d -> folded BatchNorm -> PReLU (+ residual, + x2 upsample) blocks
 * (reference: create_modules, model/models.py:49-66; shortcut add :281-282; nn.Upsample :93-94;
 *  BN folding utils/torch_utils.py:45-69).  sm_90a wgmma implicit GEMM, bf16 in / fp32 accumulate.
 *
 * Activations live in HBM as "padded NHWC": [B, H+2, W+2, Cs] bf16 with a one-pixel ZERO halo
 * (zeroed once by the owner of the buffer; these kernels never write it), channels contiguous
 * with channel stride Cs >= C, so that a 3x3/stride-1 conv is nine row-shifted GEMMs over the
 * flat pixel index and needs no im2col buffer, and channel concatenation (route layers,
 * models.py:269-278) is a write at a channel offset into a wider buffer.  Channel counts are
 * padded to multiples of 64 with zeros (the K chunk of the GEMM).
 * ------------------------------------------------------------------------------------------ */
#define RYOLO_DT_BF16 0
#define RYOLO_DT_F32 1

typedef struct ryolo_conv_desc {
  int32_t batch;       /* B                                                                   */
  int32_t in_h, in_w;  /* input spatial size (unpadded)                                       */
  int32_t cin;         /* channels read by this conv                                          */
  int32_t cin_stride;  /* channel stride of the input buffer (>= cin, multiple of 8)           */
  int32_t cout;        /* filters                                                             */
  int32_t cout_stride; /* channel stride of the bf16 output buffer (>= round_up(cout, 32); channels
                          [cout, round_up(cout,32)) are written as zeros, nothing beyond)     */
  int32_t ksize;       /* 1 or 3 (pad = (k-1)/2 as in models.py:53); 2 = 2x2 taps at offsets
                          {-1,0}^2 and -2 = offsets {0,+1}^2 (the space-to-depth form of a
                          3x3/stride-2 conv and its adjoint, see ryolo_space_to_depth)         */
  int32_t stride;      /* 1 or 2                                                              */
  int32_t has_act;     /* 1: PReLU with scalar `slope` (cfg activation=leaky), 0: linear      */
  float slope;         /* PReLU weight (nn.PReLU(num_parameters=1), models.py:65)             */
  int32_t has_residual;/* 1: add `residual` after the activation (shortcut, models.py:281-282) */
  int32_t res_stride;  /* channel stride of the residual buffer (padded NHWC at OUTPUT size)  */
  int32_t upsample2x;  /* 1: replicate each output pixel into the 2x2 block of a 2H x 2W output
                          buffer (nearest x2 folded into the producer)                        */
  int32_t out_dtype;   /* RYOLO_DT_BF16: padded NHWC; RYOLO_DT_F32: plain NCHW [B,cout,H,W]
                          (the three linear heads feeding ryolo_yolo_decode)                  */
} ryolo_conv_desc;

/* Pack reference-layout weights [cout, cin, k, k] fp32 (nn.Conv2d.weight), times an optional
 * per-filter scale (folded BN: gamma / sqrt(var + eps)), into the bf16 GEMM operand
 * [k*k][cout_pad][cin_pad] (zero padded).  Device pointers.  The operand transform is done in the
 * packing kernel (no framework-side flips / transposes / gathers): mode 0 = plain; 1 = dgrad operand
 * of a plain conv (`weight` is the FORWARD weight, `d` the dgrad descriptor: taps mirrored, matrix
 * transposed); 2 = space-to-depth form of a 3x3/stride-2 conv
 * (`weight` [cout, C, 3, 3], d->cin = 4C, d->ksize = 2); 3 = dgrad operand of mode 2 (d->cout = 4C,
 * d->ksize = -2).  ryolo_conv_unpack_wgrad is the inverse gather for weight GRADIENTS: wgrad output
 * [taps][cout_pad][cin_pad] -> nn.Conv2d layout [cout][cin][k][k] (mode 0) or, from the
 * space-to-depth form, [cout][C][3][3] (mode 2, cin = C). */
size_t ryolo_conv_packed_weight_bytes(const ryolo_conv_desc* d);
int ryolo_conv_pack_weights_ex(const ryolo_conv_desc* d, const float* weight, const float* scale,
                               void* packed_out, int mode, void* stream);
int ryolo_conv_unpack_wgrad(const float* dw, int cout_pad, int cin_pad, int mode, int cout, int cin,
                            int ksize, float* grad, void* stream);
/* Multi-tensor forms (one launch for all layers of a training step; the per-layer launches are a fixed ~2 ms per step
 * that caps strong scaling).  Job tables and prefix sums (prefix[j] = first global element of job j, prefix[njobs] =
 * total) live in DEVICE memory and are built once per plan.  Pack: `packed` receives taps*cout_pad*cin_pad bf16 for the
 * operand described like ryolo_conv_pack_weights_ex (ks = taps per side of the PACKED operand: 1, 3 or 2; cout/cin of
 * the packed operand; mode 0..3).  Unpack: `grad` receives cout*cin*ks*ks fp32 in nn.Conv2d layout (mode 0 / 2 as
 * ryolo_conv_unpack_wgrad; ks = kernel size of the nn.Conv2d weight). */
typedef struct ryolo_pack_job {
  const float* weight;
  void* packed;
  int32_t cout, cin, ks, cout_pad, cin_pad, mode;
} ryolo_pack_job;
typedef struct ryolo_unpack_job {
  const float* dw;
  float* grad;
  int32_t cout_pad, cin_pad, mode, cout, cin, ks;
} ryolo_unpack_job;
int ryolo_conv_pack_weights_multi(const ryolo_pack_job* jobs_dev, int njobs, const long long* prefix_dev,
                                  long long total, void* stream);
int ryolo_conv_unpack_wgrad_multi(const ryolo_unpack_job* jobs_dev, int njobs, const long long* prefix_dev,
                                  long long total, void* stream);
/* Zero invariants of padded-NHWC bf16 buffers [batch, h+2, w+2, c_stride] that share storage with buffers of other
 * shapes (the activation pool of a Darknet model): one launch zeroes, for every job of the table (device memory), the
 * 1-pixel halo ring (all channels) and channels [c_real, c_stride) of the interior pixels; interior channels below
 * c_real keep their bytes.  c_real = 0 zeroes the whole buffer.  ptr 16-byte aligned, c_stride % 8 == 0,
 * 0 <= c_real <= c_stride; njobs <= 65535. */
typedef struct ryolo_halo_job {
  void* ptr;
  int32_t batch, h, w, c_real, c_stride, reserved;
} ryolo_halo_job;
int ryolo_zero_halo_multi(const ryolo_halo_job* jobs_dev, int njobs, void* stream);
/* y = act(conv(x, W') + bias) [+ residual].  bias: fp32 [cout_pad] (zero beyond cout).  The implicit
 * GEMM needs no scratch memory. */
int ryolo_conv_bn_act_fwd(const ryolo_conv_desc* d, const void* x, const void* packed_w,
                          const float* bias, const void* residual, void* y, void* stream);
/* First layer (cin = 3, 3x3, stride 1; reference model/models.py:45-74 block 0): fp32 NCHW image
 * [B,3,H,W] -> bf16 padded NHWC with channel stride cout_stride (channels >= cout zero-filled).
 * weight [cout,3,3,3] fp32 with BN folded (rounded to bf16 in the kernel like every other layer's
 * weights), bias [cout], cout = 16 | 32.  The im2col row of each pixel is built in registers
 * (image split into bf16 hi + lo halves: 16 mantissa bits) and contracted with wgmma.
 * ryolo_conv_first_s2d_fwd writes the same values straight into the space-to-depth buffer of a
 * following 3x3/stride-2 layer (layout of ryolo_space_to_depth; H, W even; xs_cstride >= 4*cout). */
int ryolo_conv_first_fwd(const float* img, int batch, int h, int w, const float* weight,
                         const float* bias, int cout, float slope, void* y, int cout_stride,
                         void* stream);
int ryolo_conv_first_s2d_fwd(const float* img, int batch, int h, int w, const float* weight,
                             const float* bias, int cout, float slope, void* xs, int xs_cstride,
                             void* stream);

/* ------------------------------------------------------------------------------------------ *
 * Training path of the conv blocks (reference: autograd through nn.Conv2d / BatchNorm2d / PReLU,
 * train.py:268-282).  Same padded-NHWC bf16 layout; gradients of activations are bf16, gradients
 * of parameters fp32.
 * ------------------------------------------------------------------------------------------ */
/* dW[tap][co][ci] (fp32, [k*k][cout_pad][cin_pad], ACCUMULATED into a caller-zeroed buffer) =
 * sum over flat padded pixels p of dz[p, co] * x[p + tap_offset, ci].  dz / x: padded NHWC bf16 at
 * the conv's INPUT resolution (a stride-2 conv passes its output gradient zero-inserted onto the
 * input grid).  wgmma GEMM with K = pixels, MN-major operands, split-K
 * reduced in split order (the same dW every run). */
int ryolo_conv_wgrad(const void* dz, int dz_cstride, int cout_pad, const void* x, int x_cstride,
                     int cin_pad, int batch, int in_h, int in_w, int ksize, float* dw, void* stream);

/* Per-channel batch statistics of a raw conv output z (padded NHWC bf16, interior pixels):
 * sums[0..c) = sum z, sums[c..2c) = sum z^2 (fp32), and from them the per-channel mean, invstd,
 * scale = gamma*invstd, shift = beta - mean*scale and (when the pointers are non-null) the
 * nn.BatchNorm2d running statistics update with momentum and the unbiased variance (reference
 * model/models.py:62: momentum 0.1, eps 1e-5).  The sums are reduced in a fixed order and the
 * finalisation is fused into that reduction. */
int ryolo_bn_stats_finalize(const void* z, int z_cstride, int batch, int h, int w, int c, float* sums, float eps,
                            float momentum, const float* gamma, const float* beta, float* mean, float* invstd,
                            float* scale, float* shift, float* running_mean, float* running_var, void* stream);
/* y = prelu(z * scale + shift) [+ residual], scale/shift = folded batch-stat BN (gamma*invstd,
 * beta - mean*gamma*invstd); upsample2x writes every pixel to its 2x2 block of a 2h x 2w y. */
int ryolo_bn_act_fwd(const void* z, int z_cstride, int batch, int h, int w, int c,
                     const float* scale, const float* shift, float slope, int has_act,
                     const void* residual, int res_cstride, void* y, int y_cstride, int upsample2x,
                     const float* slope_dev, void* stream);
/* Same, and additionally writes y in the space-to-depth layout of ryolo_space_to_depth into xs (the operand of a
 * following 3x3/stride-2 block): the separate s2d pass over y disappears.  h, w even. */
int ryolo_bn_act_fwd_s2d(const void* z, int z_cstride, int batch, int h, int w, int c,
                         const float* scale, const float* shift, float slope, int has_act,
                         const void* residual, int res_cstride, void* y, int y_cstride,
                         const float* slope_dev, void* xs, int xs_cstride, void* stream);
/* slope_dev (both directions, optional): device scalar holding the PReLU slope (nn.PReLU.weight);
 * when non-null it replaces `slope`, so a training step never copies the parameter to the host.
 * Backward of the same block.  dy: gradient of y (at 2h x 2w when upsample2x == 1; upsample2x == 2: dy is read in the
 * space-to-depth layout [B, h/2+2, w/2+2, >=4c] a consuming 3x3/stride-2 block's dgrad wrote, no depth_to_space pass).  z_dz: in = z, out =
 * dz (gradient of the raw conv output, written in place).  sums (fp32 [2c+1], zeroed inside):
 * [0..c) = d(beta), [c..2c) = d(gamma), [2c] = d(slope).  gres (optional): gradient buffer of the
 * shortcut source, receives (+)= dy. */
int ryolo_bn_act_bwd(const void* dy, int dy_cstride, int upsample2x, void* z_dz, int z_cstride,
                     int batch, int h, int w, int c, const float* scale, const float* shift,
                     const float* mean, const float* invstd, float slope, int has_act, int has_bn,
                     float* sums, void* gres, int gres_cstride, int gres_accumulate,
                     const float* slope_dev, void* stream);
/* Adjoint of a stride-2 conv's pixel selection: src (h x w) -> even interior pixels of the
 * pre-zeroed dst (dst_h x dst_w). */
int ryolo_zero_insert2x(const void* src, int src_cstride, int batch, int h, int w, int c, void* dst,
                        int dst_cstride, int dst_h, int dst_w, void* stream);
/* Space-to-depth of a padded-NHWC tensor with even H, W:
 * xs[b, Y, X, (py*2+px)*C + c] = x[b, 2Y+py, 2X+px, c]  ([B, H/2+2, W/2+2, >=4C]).  A 3x3/stride-2/pad-1
 * conv on x equals a ksize=2 (offsets -1..0), stride-1 conv on xs with the weight blocks
 * W2[(qy,qx)][co][(py,px,c)] = W[co][c][kh][kw], kh = {(0,1):0,(1,0):1,(1,1):2}[(qy,py)] (zero for
 * (0,0)), same for kw.  ryolo_depth_to_space is the adjoint (optionally accumulating). */
int ryolo_space_to_depth(const void* x, int x_cstride, int batch, int h, int w, int c, void* xs,
                         int xs_cstride, void* stream);
int ryolo_depth_to_space(const void* dxs, int dxs_cstride, int batch, int h, int w, int c, void* gx,
                         int gx_cstride, int accumulate, void* stream);
/* Phase decomposition of a dilated 3x3 conv (reference `[d-convolutional]` blocks: F.conv2d with dilation (dh, dw),
 * pad (dh, dw), model/models.py:262-265).  ryolo_dilate_split writes the dh*dw phase images of x ([B, H+2, W+2, >=C])
 * into xp ([B*dh*dw, Hp+2, Wp+2, >=C], Hp = ceil(H/dh), Wp = ceil(W/dw), zero halo):
 *   xp[(b*dh + ry)*dw + rx, Y, X, c] = x[b, Y*dh + ry, X*dw + rx, c], 0 where Y*dh + ry >= H or X*dw + rx >= W.
 * On xp the dilated conv is an ordinary pad-1 3x3 conv with batch B*dh*dw.  ryolo_dilate_merge writes the interior of
 * y back from the phase images: y[b, y, x, c] = xp[phase of (y, x)] (+ residual[b, y, x, c]) (+ y[b, y, x, c] when
 * accumulate), summed in fp32 in that order and rounded to bf16 once.  Each is the other's adjoint.  C % 8 == 0,
 * channel strides % 8 == 0, 16-byte aligned pointers.  The extents are not checked: xp must hold
 * [B*dh*dw, Hp+2, Wp+2, xp_cstride] (x and y [B, H+2, W+2, their cstride]), and xp's halo must already be zero -- the
 * split writes the interior (zero fill included) and channels [0, C) only; the merge writes y's interior only. */
int ryolo_dilate_split(const void* x, int x_cstride, int batch, int h, int w, int c, int dh, int dw, void* xp,
                       int xp_cstride, void* stream);
int ryolo_dilate_merge(const void* xp, int xp_cstride, int batch, int h, int w, int c, int dh, int dw,
                       const void* residual, int res_cstride, int accumulate, void* y, int y_cstride, void* stream);
/* Squeeze-and-excitation block (reference SELayer, model/models.py:16-31; `[se]` blocks of cfg/ICDAR/yolov3_608_se.cfg,
 * cfg/HRSC+/yolov3_512_se.cfg): x[b,:,:,c] *= sigmoid(W2 . relu(W1 . mean_hw x[b]))[c], in place on a padded-NHWC bf16
 * tensor.  w1 [reduced, c], w2 [c, reduced] fp32 (nn.Linear weights, no bias); sums_scratch / scale_scratch [batch*c]
 * fp32.  Eval path. */
int ryolo_se_block(void* x, int x_cstride, int batch, int h, int w, int c, const float* w1, const float* w2,
                   int reduced, float* sums_scratch, float* scale_scratch, void* stream);
/* The same block out of place and deterministic, for graphs whose SE input x is read again (the reference's *_se.cfg: the
 * shortcut three blocks later adds x, concat routes read x) and for training.  Per image b, channel c:
 *   m = mean_hw x,  p = W1 m,  s = sigmoid(W2 relu(p)),  u = bf16(x s)  (u's halo is not written).
 * m, s [batch, c] and p [batch, reduced] fp32 are outputs the backward reads.  Backward, gu = dL/du:
 *   ds = sum_hw gu x,  da = ds s (1 - s),  dhid = (W2^T da) [p > 0],  dm = W1^T dhid,
 *   gx = bf16([gx +] gu s + dm / hw)  (accumulate = 1 adds to the gradient other writers left in gx),
 *   gw1 = sum_b dhid m^T [reduced, c],  gw2 = sum_b da relu(p)^T [c, reduced]  (overwritten; fp32).
 * ds, dm [batch, c] fp32 are outputs.  Every reduction runs in a fixed order, none uses float atomics; an image's
 * results do not depend on the batch it is in.  c % 8 == 0, c <= 2048; x, u, gu, gx 16-byte aligned.  workspace
 * (caller-owned, >= ryolo_se_workspace_bytes) serves both directions; no allocation, no host synchronisation. */
size_t ryolo_se_workspace_bytes(int batch, int h, int w, int c, int reduced);
int ryolo_se_fwd(const void* x, int x_cstride, void* u, int u_cstride, int batch, int h, int w, int c,
                 const float* w1, const float* w2, int reduced, float* m, float* p, float* s, void* workspace,
                 size_t workspace_bytes, void* stream);
int ryolo_se_bwd(const void* gu, int gu_cstride, const void* x, int x_cstride, void* gx, int gx_cstride,
                 int accumulate, int batch, int h, int w, int c, const float* w1, const float* w2, int reduced,
                 const float* m, const float* p, const float* s, float* ds, float* dm, float* gw1, float* gw2,
                 void* workspace, size_t workspace_bytes, void* stream);
/* 2x2 max pooling of a padded-NHWC bf16 tensor (reference: the maxpool blocks of
 * cfg/yolov3-tiny.cfg, model/models.py:79-87).  stride 2: [in_h/2, in_w/2] output; stride 1: same
 * size, the window past the right/bottom edge reads the zero halo exactly like the reference's
 * nn.ZeroPad2d((0,1,0,1)) + MaxPool2d(2, 1). */
int ryolo_maxpool2x2(const void* x, int x_cstride, int batch, int in_h, int in_w, int c, int stride,
                     void* y, int y_cstride, void* stream);
/* Gradient of a YOLO head -> bf16 padded NHWC [B, ny+2, nx+2, dst_cstride], channels >= C and the halo left
 * untouched.  The cotangent is in the layout the head convolution WROTE its output in: fp32 NCHW [B, C = na*no, ny, nx]
 * (what arrives when the consumer differentiates the permuted VIEW of that buffer, e.g. the fused loss below).
 * bias_grad (nullable): [C] fp32, the per-channel sums of g are ADDED to it (the head convolution's bias gradient);
 * C <= 2048. */
int ryolo_head_grad_nchw_to_padded(const float* g, int batch, int c, int ny, int nx, void* dst,
                                   int dst_cstride, float* bias_grad, void* stream);
/* The bias gradient alone of the same cotangent: the per-channel sums of g are ADDED to bias_grad ([C] fp32), in the
 * same order as ryolo_head_grad_nchw_to_padded takes them, so the same bits; g is read once and nothing else is written
 * (training with the head convolution's weight and everything below it frozen); C <= 2048. */
int ryolo_head_bias_grad(const float* g, int batch, int c, int ny, int nx, float* bias_grad, void* stream);
/* Objectness term of compute_loss (reference model/loss.py:340-348: BCEWithLogitsLoss(pos_weight)(pi[..., 5], tobj)
 * over every cell of a head map).  x: logical [batch, na, ny, nx, no] fp32 tensor addressed through `strides` (5 element
 * strides, so both the contiguous tensor and the permuted view of the NCHW head buffer are read in place); ch = the
 * objectness channel; tobj: contiguous [batch, na, ny, nx].  fwd ADDS the sum of the element losses to *sum_out
 * (float64, caller zeroes it and divides by the cell count); bwd writes the whole cotangent tensor `grad` (strides of x):
 * channel ch = *scale_dev * d(loss)/dx, every other channel 0. */
int ryolo_obj_bce_fwd(const float* x, const long long* strides, int batch, int na, int ny, int nx, int no, int ch,
                      const float* tobj, float pos_weight, double* sum_out, void* stream);
int ryolo_obj_bce_bwd(const float* x, const long long* strides, int batch, int na, int ny, int nx, int no, int ch,
                      const float* tobj, float pos_weight, const float* scale_dev, float* grad, void* stream);
/* Focal form of the same term (arcs containing 'F', reference model/loss.py:126-146, 284-286): per cell the BCE loss l
 * becomes l * (1.000001 - exp(-l))^gamma (alpha = 1), the factor evaluated as (2^-20 - expm1(-l))^gamma.  Arguments and
 * outputs as ryolo_obj_bce_*, plus gamma (finite, >= 0); gamma = 0 gives the bits of ryolo_obj_bce_*. */
int ryolo_obj_focal_fwd(const float* x, const long long* strides, int batch, int na, int ny, int nx, int no, int ch,
                        const float* tobj, float pos_weight, float gamma, double* sum_out, void* stream);
int ryolo_obj_focal_bwd(const float* x, const long long* strides, int batch, int na, int ny, int nx, int no, int ch,
                        const float* tobj, float pos_weight, float gamma, const float* scale_dev, float* grad,
                        void* stream);
/* The matched (anchor, target) rows of compute_loss (reference model/loss.py:300-338 indexes `pi[b, a, gj, gi]`): int64
 * device index vectors b / a / gj / gi and a 0/1 byte mask, `rows` entries each.  gather: out[r, k] = x[b, a, gj, gi, k]
 * (0 for masked-out or out-of-range rows); set_tobj: tobj[b, a, gj, gi] = 1 (tobj contiguous [batch, na, ny, nx]);
 * scatter_add: grad[b, a, gj, gi, k] += vals[r, k] * *scale_dev (duplicated cells accumulate like autograd's
 * index backward, in row order).  x / grad are addressed through 5 element strides like ryolo_obj_bce_*. */
int ryolo_loss_rows_gather(const float* x, const long long* strides, int batch, int na, int ny, int nx, int no,
                           const long long* b, const long long* a, const long long* gj, const long long* gi,
                           const unsigned char* mask, int rows, float* out, void* stream);
int ryolo_loss_rows_scatter_add(float* grad, const long long* strides, int batch, int na, int ny, int nx, int no,
                                const long long* b, const long long* a, const long long* gj, const long long* gi,
                                const unsigned char* mask, int rows, const float* vals, const float* scale_dev,
                                void* stream);
int ryolo_loss_rows_set_tobj(float* tobj, int batch, int na, int ny, int nx, const long long* b, const long long* a,
                             const long long* gj, const long long* gi, const unsigned char* mask, int rows, void* stream);
/* im2col of the 3-channel fp32 image for the first 3x3 conv: bf16 padded NHWC with 64 channels
 * (27 real, column = c*9 + kh*3 + kw), so that the first layer runs on the same GEMM kernels. */
int ryolo_im2col_first(const float* img, int batch, int h, int w, void* dst, void* stream);

/* ------------------------------------------------------------------------------------------ *
 * Parity-precision path (Darknet(..., precision="parity")): fp32-grade conv blocks on the bf16
 * tensor pipe, for the 1e-4 tolerance north_star states against the reference's fp32 nn.Conv2d
 * (model/models.py:55-65).  GEMM operands are SPLIT bf16 tensors: padded NHWC like above, but
 * every value v is two planes hi = bf16(v), lo = bf16(v - hi), `lo` channels apart in the same
 * row ("split view": pointer to channel 0 of plane 0, channel stride, plane offset `lo`, number of
 * planes: plane k = bf16 of the remainder left by planes < k, k*lo channels further; three planes
 * carry all 24 bits of an fp32).  Conv results, BN / PReLU / shortcut arithmetic and all gradients
 * of activations are fp32 padded NHWC; reductions are fp64.  a*w is evaluated as a sum of TERMS
 * a_i*w_j (a term table, 2 bits per term per operand: i + j <= 2 for three planes), exact products;
 * the wgmma accumulator is restarted every 8 k-steps and folded into round-to-nearest fp32 register sums
 * (the tensor pipe's own accumulator does not round to nearest, DESIGN.md).
 * ------------------------------------------------------------------------------------------ */
/* weight [cout,cin,k,k] fp32 -> bf16 [k*k][round_up(cout,64)][nterms*round_up(cin,64)]; term t of the
 * K range holds plane (w_plane_code >> 2t) & 3.  mode as ryolo_conv_pack_weights_ex
 * (ksize 2 / -2 for the space-to-depth forms; cout/cin are those of the PACKED operand). */
size_t ryolo_px_packed_weight_bytes(int cout, int cin, int ksize, int nterms);
int ryolo_px_pack_weights(const float* weight, int cout, int cin, int ksize, int nterms,
                          int w_plane_code, int mode, void* packed_out, void* stream);
/* out[p, co] (+)= sum over terms, taps, channels.  x_base: start of the split buffer row 0, the view
 * starts x_ch_off channels in; (a_plane_code >> 2t) & 3 is the activation plane of term t.  out: fp32
 * padded NHWC on the same grid (stride 1; stride-2 convs run on space-to-depth inputs), columns
 * [0, out_cols) written, accumulate != 0 adds to the existing contents (dgrad). */
int ryolo_px_conv(const void* x_base, int x_cstride, int x_ch_off, int plane_stride, int cin,
                  const void* packed_w, int nterms, int a_plane_code, int batch, int in_h, int in_w,
                  int ksize, int cout, float* out, int out_cstride, int out_cols, int accumulate,
                  void* stream);
/* wgrad of split operands = ryolo_px_wgrad over all planes of dz and x ([taps][np*plane_out][np*plane_in]);
 * this sums the nplanes^2 plane blocks into nn.Conv2d layout (mode 0 / 2 as ryolo_conv_unpack_wgrad); cin_off:
 * first channel of x's view inside its plane (a conv reading a slice of a concat buffer). */
int ryolo_px_unpack_wgrad(const float* dw, int plane_out, int plane_in, int nplanes, int mode, int cout,
                          int cin, int ksize, int cin_off, float* grad, void* stream);
/* ryolo_conv_wgrad with the accumulation of ryolo_px_conv: the wgmma accumulator is restarted every 8
 * k-steps and folded into round-to-nearest fp32 register sums, so the dW of a long pixel range carries no
 * truncation bias.  Same arguments and dW layout; the parity path runs it over all planes of dz and x. */
int ryolo_px_wgrad(const void* dz, int dz_cstride, int cout_pad, const void* x, int x_cstride,
                   int cin_pad, int batch, int in_h, int in_w, int ksize, float* dw, void* stream);
/* batch statistics of fp32 z: sums[0..c) = sum, [c..2c) = sum of squares (fp64, zeroed inside) */
int ryolo_px_bn_stats(const float* z, int z_cstride, int batch, int h, int w, int c, double* sums,
                      void* stream);
/* eval_mode 0: batch statistics from sums (running statistics updated); 1: running statistics. */
int ryolo_px_bn_finalize(const double* sums, int c, double count, float eps, float momentum,
                         const float* gamma, const float* beta, int eval_mode, float* mean,
                         float* invstd, float* scale, float* shift, float* running_mean,
                         float* running_var, void* stream);
/* y = prelu(z*scale + shift) [+ residual] -> split view (slope_dev NULL: linear) */
int ryolo_px_bn_act_fwd(const float* z, int z_cstride, int batch, int h, int w, int c,
                        const float* scale, const float* shift, const float* slope_dev,
                        const void* residual, int res_cstride, int res_lo, void* y, int y_cstride,
                        int y_lo, int upsample2x, int nplanes, void* stream);
/* backward: dy fp32 (2h x 2w when upsample2x), z fp32 -> sums fp64 [2c+1] (d beta, d gamma, d slope),
 * dz split view, shortcut gradient gres fp32 (+)= dy. */
int ryolo_px_bn_act_bwd(const float* dy, int dy_cstride, int upsample2x, const float* z, int z_cstride,
                        int batch, int h, int w, int c, const float* scale, const float* shift,
                        const float* mean, const float* invstd, const float* slope_dev,
                        int batch_stats, double* sums, void* dz, int dz_cstride, int dz_lo, float* gres,
                        int gres_cstride, int gres_accumulate, int nplanes, void* stream);
int ryolo_px_im2col_first(const float* img, int batch, int h, int w, void* dst, int dst_cstride,
                          int dst_lo, int nplanes, void* stream);
/* fp32 padded NHWC (+ bias[c]) -> fp32 NCHW [B,c,h,w] (the linear heads feeding ryolo_yolo_decode) */
int ryolo_px_to_nchw(const float* z, int z_cstride, int batch, int c, int h, int w, const float* bias,
                     float* out, void* stream);
int ryolo_px_head_grad(const float* g, int batch, int na, int no, int ny, int nx, void* dst,
                       int dst_cstride, int dst_lo, int nplanes, void* stream);
int ryolo_px_depth_to_space(const float* dxs, int dxs_cstride, int batch, int h, int w, int c, float* gx,
                            int gx_cstride, int accumulate, void* stream);
int ryolo_px_split_from_nchw(const float* src, int batch, int c, int h, int w, void* dst,
                             int dst_cstride, int dst_lo, int nplanes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Letterbox <- letterbox()                               utils/datasets.py:512-546
 *              LoadImages / LoadImagesAndLabels normalisation   utils/datasets.py:112-117, 498-500
 * One launch letterboxes a batch of uint8 HWC BGR images of any sizes into out [njobs, 3, out_h, out_w]
 * (RGB, value/255 by IEEE division, fp32 or fp16; border pixels 128/255), byte for byte what
 * cv2.resize(INTER_AREA) + copyMakeBorder + the reference's normalisation compute.  jobs_dev and tables_dev
 * are device memory built from shapes alone (rotate-yolov3_b200/preprocess.py).  A job's per-axis table at
 * word offset xtab / ytab of tables_dev holds, per output index d, three int32 {start, count, woff}: the taps
 * are source indices start + t (t < count; clipped to the image for RYOLO_LB_LINEAR) with weights at word
 * offset xtab + woff (float32 for RYOLO_LB_AREA, int32 for RYOLO_LB_LINEAR, none for RYOLO_LB_AREA_INT).
 * No resize is RYOLO_LB_AREA with one unit tap per pixel.  Requires top + dst_h <= out_h,
 * left + dst_w <= out_w; njobs <= 65535.  Allocates nothing; capturable in a CUDA graph.
 * out_dtype RYOLO_DT_U8 writes the letterboxed uint8 image instead: out [njobs, out_h, out_w, 3] BGR, border 128
 * (the training augmentation's intermediate; with top = left = 0 it is a plain batched resize).
 * ------------------------------------------------------------------------------------------ */
#define RYOLO_DT_F16 2
#define RYOLO_DT_U8 3
#define RYOLO_LB_AREA 0     /* float32 area weights (non-integer downscale, or a copy)          */
#define RYOLO_LB_AREA_INT 1 /* integer factors kx x ky: integer sums                             */
#define RYOLO_LB_LINEAR 2   /* an axis upscales: 2-tap linear, 11-bit fixed-point weights        */
typedef struct ryolo_letterbox_job {
  const uint8_t* src;  /* [src_h, src_w, 3] BGR, pixels contiguous                            */
  int64_t src_stride;  /* bytes between source rows                                           */
  int32_t src_h, src_w;
  int32_t dst_h, dst_w; /* resized (unpadded) size                                            */
  int32_t top, left;    /* border above / left of the resized image                            */
  int32_t kind;         /* RYOLO_LB_*                                                          */
  int32_t kx, ky;       /* RYOLO_LB_AREA_INT factors                                           */
  int32_t xtab, ytab;   /* word offsets of the per-axis tables in tables_dev                   */
  int32_t reserved;
} ryolo_letterbox_job;
int ryolo_letterbox(const ryolo_letterbox_job* jobs_dev, int njobs, const int32_t* tables_dev, void* out,
                    int out_h, int out_w, int out_dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * Training augmentation <- utils/augment.py random_affine, Gamma, HSV, HorizontalFlip, VerticalFlip
 *                          and the LoadImagesAndLabels normalisation   utils/datasets.py:470-500
 * Both launches run over a batch of letterboxed uint8 [h, w, 3] BGR images (ryolo_letterbox with RYOLO_DT_U8).
 *
 * ryolo_augment_warp: one job per image that is warped or whose maximum gamma needs.  warp = 1:
 *   cv2.warpAffine(src, M, (w, h), INTER_LINEAR, border 128) into dst [h, w, 3] (rows of 3 * w bytes), given m,
 *   the inverse of M as cv2 inverts it; cv2's fixed-point remap (10-bit AB, 5-bit INTER fractions, 15-bit
 *   weights).  rowmax[image * h + y] = max over row y of dst (warp = 1) or of src (warp = 0, dst unused).
 * ryolo_augment_finish: one job per image, job b writes out[b] [3, h, w] (RGB, /255, fp32 or fp16) from src
 *   (the warped or letterboxed image): gamma uint8(pow(v / M, gamma) * M) with M = max of rowmax[b * h ..
 *   b * h + h) (0 when M = 0), then cv2's 8-bit BGR2HSV, S and V scaled by the float32 factors and truncated,
 *   8-bit HSV2BGR, then the flips, each when its flag is set.
 * njobs <= 65535.  Allocate nothing; capturable in a CUDA graph.
 * ------------------------------------------------------------------------------------------ */
#define RYOLO_AUG_GAMMA 1
#define RYOLO_AUG_HSV 2
#define RYOLO_AUG_HFLIP 4
#define RYOLO_AUG_VFLIP 8
typedef struct ryolo_warp_job {
  const uint8_t* src;  /* [h, w, 3] BGR, rows of src_stride bytes                                */
  uint8_t* dst;        /* [h, w, 3] BGR, rows of 3 * w bytes (warp = 1)                          */
  int64_t src_stride;
  double m[6];         /* dst -> src affine map, row major 2 x 3                                 */
  int32_t warp;        /* 1: warp into dst and take its row maxima; 0: row maxima of src only   */
  int32_t image;       /* row block of rowmax                                                    */
} ryolo_warp_job;
typedef struct ryolo_finish_job {
  const uint8_t* src;  /* [h, w, 3] BGR, rows of src_stride bytes                                */
  int64_t src_stride;
  double gamma;        /* RYOLO_AUG_GAMMA exponent                                               */
  float hsv_s, hsv_v;  /* RYOLO_AUG_HSV factors, >= 0                                            */
  int32_t flags;       /* RYOLO_AUG_*                                                            */
  int32_t reserved;
} ryolo_finish_job;
int ryolo_augment_warp(const ryolo_warp_job* jobs_dev, int njobs, uint8_t* rowmax, int h, int w, void* stream);
int ryolo_augment_finish(const ryolo_finish_job* jobs_dev, int njobs, const uint8_t* rowmax, void* out, int h, int w,
                         int out_dtype, void* stream);

/* ------------------------------------------------------------------------------------------
 * JPEG decode <- cv2.imread(path) (IMREAD_COLOR)          utils/datasets.py:105, 382, 434
 * Decodes a batch of 8-bit sequential Huffman JPEG streams with one interleaved scan (1 or 3 components,
 * sampling 4:4:4, 4:2:2, 4:2:0, 4:4:0, 4:1:1) into uint8 HWC BGR images, byte for byte what libjpeg-turbo's
 * default decompression computes (ISLOW IDCT, fancy upsampling, YCbCr -> BGR), with the Exif orientation
 * applied as cv2.imread applies it.  The host parses the markers and builds the tables
 * (rotate-yolov3_b200/decode.py); csrc/jpeg.cuh holds the per-symbol and per-pixel arithmetic.
 *
 * Entropy decoding runs per restart interval (a segment: the bytes [start, end) between markers), split into
 * chunks of chunk_bytes, one thread per chunk (Weissenberger & Schmidt, ICPP 2018): each chunk is decoded from
 * its first byte, then each thread decodes on from where the previous chunk's decoder stopped until its state
 * (bit position, coefficient index, block within the MCU) matches the state the chunk decoder reached at the same
 * chunk end, and the chunks on the true decode path write the coefficients.
 * chunk_seg[c] is chunk c's segment; a segment's chunks are consecutive (first_chunk .. first_chunk + nchunk).
 * huff holds the Huffman tables the images refer to, quant 64 quantisation values per table in natural order.
 * max_blocks >= blocks of any image (mcux * mcuy * bpm), max_out_h >= out rows of any image.
 * status[i] is set to a nonzero RYOLO_JPEG_ST_* mask when image i cannot be decoded on the device (a code not
 * in its table, a coefficient run past the block, data ending before the last block, a chunk that does not
 * synchronise, a block whose dequantised coefficients or samples leave the range where libjpeg-turbo's C and SIMD
 * IDCTs agree); its output is then unspecified.  Every read stays inside its segment.  The pixel stage adds its
 * bit to what the entropy stage left in status.
 * stages: RYOLO_JPEG_ENTROPY (status, coefficients), RYOLO_JPEG_PIXELS (IDCT, upsampling, colour, store) or both;
 * the second reads the coefficients the first left in the workspace.  image_bytes: the size of the image area
 * the images' coef_off / plane_off point into.  Allocates nothing; capturable in a CUDA graph; data < 4 GiB.
 * ------------------------------------------------------------------------------------------ */
#define RYOLO_JPEG_YCC 0         /* YCbCr -> BGR                                                        */
#define RYOLO_JPEG_RGB 1         /* stored as RGB (Adobe transform 0 or component ids 'R', 'G', 'B')    */
#define RYOLO_JPEG_GRAY 2        /* one component, replicated into B, G, R                             */
#define RYOLO_JPEG_ENTROPY 1
#define RYOLO_JPEG_PIXELS 2
#define RYOLO_JPEG_ST_BAD_CODE 1  /* a code not in its table, or a run past coefficient 63          */
#define RYOLO_JPEG_ST_TRUNCATED 2 /* the segment ends before its last block                         */
#define RYOLO_JPEG_ST_NO_SYNC 4   /* a chunk on the decode path did not synchronise                 */
#define RYOLO_JPEG_ST_RANGE 8     /* a block outside the range where every libjpeg-turbo IDCT agrees  */
typedef struct ryolo_jpeg_image {
  int64_t out_off;      /* byte offset of the [out_h, out_w, 3] BGR image in out                              */
  int64_t coef_off;     /* byte offset in the image area of the int16 coefficient blocks, in decode order      */
  int64_t plane_off[3]; /* byte offsets in the image area of the component sample planes                      */
  int32_t width, height;  /* stored size                                                                   */
  int32_t out_w, out_h;   /* size after the orientation                                                    */
  int32_t orient;         /* Exif orientation 1..8                                                         */
  int32_t ncomp, color;   /* 1 or 3; RYOLO_JPEG_YCC / RGB / GRAY                                           */
  int32_t hmax, vmax;     /* largest sampling factors                                                      */
  int32_t mcux, mcuy, bpm; /* MCUs per row, MCU rows, blocks per MCU                                       */
  int32_t h[3], v[3];     /* sampling factors                                                              */
  int32_t boff[3];        /* first block of the component within the MCU (64 for absent components)        */
  int32_t pitch[3];       /* plane row bytes, mcux * h * 8 (rows: mcuy * v * 8)                            */
  int32_t dw[3], dh[3];   /* component size, ceil(width * h / hmax) x ceil(height * v / vmax)              */
  int32_t qtab[3];        /* first value of the component's quantisation table in quant                    */
  int32_t dctab[3], actab[3]; /* the component's Huffman tables in huff                                    */
  int32_t reserved;
} ryolo_jpeg_image;
typedef struct ryolo_jpeg_segment {
  int64_t start, end;      /* entropy-coded bytes [start, end) in data, stuffing included                       */
  int32_t image, first_mcu, nmcu;
  int32_t first_chunk, nchunk;
  int32_t reserved;
} ryolo_jpeg_segment;
typedef struct ryolo_jpeg_huff {
  uint16_t lut[512];    /* 9-bit lookahead: (length << 8) | symbol, 0 when the code is longer than 9 bits       */
  int32_t maxcode[18];  /* largest code of each length, -1 when there is none (libjpeg's derived table)          */
  int32_t valoff[18];   /* symbol index minus code, per length                                                  */
  uint8_t vals[256];    /* symbols in code order                                                                */
} ryolo_jpeg_huff;
size_t ryolo_jpeg_workspace_bytes(int nchunks, long long image_bytes);
int ryolo_jpeg_decode(const ryolo_jpeg_image* images, int nimages, const ryolo_jpeg_segment* segs, int nsegs,
                      const int32_t* chunk_seg, int nchunks, int chunk_bytes, const uint8_t* data,
                      long long data_bytes, const ryolo_jpeg_huff* huff, const uint16_t* quant, int max_blocks,
                      int max_out_h, uint8_t* out, int32_t* status, void* workspace, size_t workspace_bytes,
                      long long image_bytes, int stages, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RYOLO_H_ */
