/*
 * vision_b200.h — C ABI of libvision_b200.so (sm_90a CUDA kernels for the
 * torchvision custom-op hot path).  No torch types cross this boundary: plain
 * device pointers, sizes and a CUDA stream handle.  Every entry point names
 * the reference interface it replaces (paths relative to pytorch/vision).
 *
 * Conventions
 *   - all data pointers are DEVICE pointers unless the name ends in `_host`;
 *   - tensors are dense, row-major ("contiguous") NCHW exactly as the
 *     reference kernels receive them after `.contiguous()`;
 *   - `stream` is a cudaStream_t passed as void*; work is enqueued on it and
 *     the call returns without synchronising unless documented otherwise;
 *   - return value: 0 on success, otherwise a negative VB200_E* code or a
 *     positive cudaError_t; vb200_last_error() gives a thread-local message
 *     (the torch shim turns it into the RuntimeError the reference raises).
 */
#ifndef VISION_B200_H_
#define VISION_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VB200_ABI_VERSION 2

#if defined(__GNUC__)
#define VB200_API __attribute__((visibility("default")))
#else
#define VB200_API
#endif

typedef enum {
  VB200_F32 = 0,
  VB200_F16 = 1,
  VB200_BF16 = 2,
  VB200_F64 = 3,
  VB200_U8 = 4
} vb200_dtype;

enum {
  VB200_OK = 0,
  VB200_EINVAL = -1,      /* bad argument (shape / dtype / alignment) */
  VB200_EUNSUPPORTED = -2,/* valid request this build does not implement */
  VB200_EWORKSPACE = -3   /* workspace too small */
};

/* NMS IoU arithmetic selector.  VB200_NMS_CUDA reproduces the compiled
 * reference CUDA kernel (csrc/ops/cuda/nms_kernel.cu:42-54: Sb's product is
 * FMA-contracted into Sa+Sb, threshold narrowed to float); VB200_NMS_CPU
 * reproduces csrc/ops/cpu/nms_kernel.cpp:58,78-88 (separately rounded areas,
 * comparison against the double threshold). */
enum { VB200_NMS_CPU = 0, VB200_NMS_CUDA = 1 };

/* batched_nms strategy (torchvision/ops/boxes.py:86-89). AUTO applies the
 * reference's own switch for CUDA tensors (numel > 100_000 -> VANILLA). */
enum { VB200_BNMS_AUTO = 0, VB200_BNMS_VANILLA = 1, VB200_BNMS_TRICK = 2 };
/* OR-ed into `strategy`: sort class ids as full 64-bit keys.  Without it the per-class path
 * speculates that ids lie in [0, 65536) (2 radix passes instead of 8); if they do not, the call
 * reports *num_keep_out = -1 and must be repeated with this flag. */
#define VB200_BNMS_WIDE_KEYS 0x100

enum { VB200_RESIZE_BILINEAR = 0, VB200_RESIZE_BICUBIC = 1 };

typedef void* vb200_stream; /* cudaStream_t */

VB200_API int vb200_abi_version(void);
VB200_API const char* vb200_last_error(void);
/* Number of kernel launches issued by this library in this process (all
 * threads); bench.py reports the delta over the timed region. */
VB200_API uint64_t vb200_launch_count(void);
/* The VB200_* path overrides (DESIGN.md, testing / profiling only) are read from the environment once, the first
 * time a launcher needs them; this re-reads them (tests switch paths inside one process). */
VB200_API void vb200_reload_env(void);

/* ---- roi_align ---------------------------------------------------------
 * Replaces roi_align_forward_kernel, csrc/ops/cuda/roi_align_kernel.cu:334-394
 * (schema torchvision::roi_align, csrc/ops/roi_align.cpp:74-75).
 * input [batch, channels, height, width], rois [num_rois, 5] (same dtype),
 * output [num_rois, channels, pooled_h, pooled_w] — written in full, no
 * pre-zeroing needed.  dtype: F32, F16, F64.
 * workspace: vb200_roi_align_workspace_bytes() bytes of device scratch (the
 * per-RoI sampling geometry of the plane-resident path; 0 when not needed). */
VB200_API size_t vb200_roi_align_workspace_bytes(int dtype, int batch, int channels, int height, int width,
                                       int num_rois, int pooled_h, int pooled_w,
                                       int sampling_ratio);
VB200_API int vb200_roi_align_forward(const void* input, const void* rois, void* output, int dtype,
                            int batch, int channels, int height, int width, int num_rois,
                            int pooled_h, int pooled_w, double spatial_scale,
                            int sampling_ratio, int aligned, void* workspace,
                            size_t workspace_bytes, vb200_stream stream);
/* roi_align fused with the all-gather of its output over the GPUs of one box (SURVEY.md 8e): outputs[0] is the caller's slot
 * of its own gathered buffer, outputs[1..n_outputs) the SAME slot of every peer's buffer (peer-mapped device pointers);
 * multicast_output, when not NULL, is ONE NVSwitch multicast address of that slot and replaces the per-peer stores
 * (multimem.st: the switch replicates each store to every rank, the local one included; fp32 only).  Same arguments and
 * workspace as vb200_roi_align_forward otherwise.  The caller synchronises the ranks before anyone reads the buffers. */
VB200_API int vb200_roi_align_forward_gather(const void* input, const void* rois, void* const* outputs, int n_outputs,
                                   void* multicast_output, int dtype, int batch, int channels, int height, int width,
                                   int num_rois, int pooled_h, int pooled_w, double spatial_scale, int sampling_ratio,
                                   int aligned, void* workspace, size_t workspace_bytes, vb200_stream stream);

/* ---- MultiScaleRoIAlign, fused -----------------------------------------
 * Replaces _multiscale_roi_align, torchvision/ops/poolers.py:147-228: per level {where, gather rois, roi_align,
 * scatter into a zeroed result} plus the LevelMapper (poolers.py:47-84) as a chain of tensor ops - here ONE geometry
 * launch (LevelMapper evaluated on the device, RoIs bucketed by level) and ONE gather launch whose work list runs over
 * the channel planes of every level; output rows are written in place (no zero-fill, no scatter).
 * level_ptrs / heights / widths / scales: HOST arrays of num_levels entries (device pointers of [batch, channels, H_l, W_l]
 * fp32 maps); rois [num_rois, 5] (batch index, x1, y1, x2, y2 in image coordinates); output [num_rois, channels, 7, 7];
 * levels_out [num_rois] int32 = level index of every RoI (for the backward pass).  aligned = False as the reference
 * calls it.  Supported: fp32, 7x7 bins, sampling_ratio 2, <= 8 levels, every plane fits shared memory
 * (vb200_multiscale_roi_align_supported); other configurations stay on the per-level path. */
VB200_API size_t vb200_multiscale_roi_align_workspace_bytes(int num_rois, int num_levels);
VB200_API int vb200_multiscale_roi_align_supported(int dtype, int num_levels, const int* heights, const int* widths,
                                         int pooled_h, int pooled_w, int sampling_ratio);
VB200_API int vb200_multiscale_roi_align_forward(const void* const* level_ptrs, const int* heights, const int* widths,
                                       const double* scales, int num_levels, const void* rois, void* output,
                                       int32_t* levels_out, int dtype, int batch, int channels, int num_rois,
                                       int pooled_h, int pooled_w, int sampling_ratio, int k_min, int k_max,
                                       double canonical_scale, double canonical_level, double eps, void* workspace,
                                       size_t workspace_bytes, vb200_stream stream);

/* ---- roi_pool ----------------------------------------------------------
 * Replaces roi_pool_forward_kernel, csrc/ops/cuda/roi_pool_kernel.cu:127-188
 * (schema torchvision::roi_pool, csrc/ops/roi_pool.cpp:67-68).
 * argmax [num_rois, channels, pooled_h, pooled_w] int32. */
VB200_API int vb200_roi_pool_forward(const void* input, const void* rois, void* output, int32_t* argmax,
                           int dtype, int batch, int channels, int height, int width,
                           int num_rois, int pooled_h, int pooled_w, double spatial_scale,
                           vb200_stream stream);

/* ---- ps_roi_align ------------------------------------------------------
 * Replaces ps_roi_align_forward_kernel, csrc/ops/cuda/ps_roi_align_kernel.cu:319-389
 * (schema torchvision::ps_roi_align, csrc/ops/ps_roi_align.cpp:74-75).
 * channels must be a multiple of pooled_h*pooled_w; output and
 * channel_mapping are [num_rois, channels/(pooled_h*pooled_w), pooled_h, pooled_w]. */
VB200_API int vb200_ps_roi_align_forward(const void* input, const void* rois, void* output,
                               int32_t* channel_mapping, int dtype, int batch, int channels,
                               int height, int width, int num_rois, int pooled_h, int pooled_w,
                               double spatial_scale, int sampling_ratio, vb200_stream stream);

/* ---- ps_roi_pool (API completeness, SURVEY.md §8f4) --------------------
 * Replaces ps_roi_pool_forward_kernel / ps_roi_pool_backward_kernel, csrc/ops/cuda/ps_roi_pool_kernel.cu:15-142
 * (schemas csrc/ops/ps_roi_pool.cpp:71-73).  Shapes as ps_roi_align; the backward writes grad_input in full itself.
 * With deterministic == 0 (workspace unused) the backward is an atomic scatter; with deterministic != 0 and
 * vb200_roi_backward_workspace_bytes(num_rois, pooled_h, pooled_w, 1) bytes of workspace it is bit-reproducible (see the
 * backward section below). */
VB200_API int vb200_ps_roi_pool_forward(const void* input, const void* rois, void* output, int32_t* channel_mapping, int dtype,
                              int batch, int channels, int height, int width, int num_rois, int pooled_h, int pooled_w,
                              double spatial_scale, vb200_stream stream);
VB200_API int vb200_ps_roi_pool_backward(const void* grad, const void* rois, void* grad_input, int dtype, int batch, int channels,
                               int height, int width, int num_rois, int pooled_h, int pooled_w, double spatial_scale,
                               int deterministic, void* workspace, size_t workspace_bytes, vb200_stream stream);

/* ---- backward of the RoI ops --------------------------------------------
 * Replace roi_align_backward_kernel (csrc/ops/cuda/roi_align_kernel.cu:396-468, schema roi_align.cpp:76-77),
 * roi_pool_backward_kernel (cuda/roi_pool_kernel.cu:190-260, schema roi_pool.cpp:69-70) and
 * ps_roi_align_backward_kernel (cuda/ps_roi_align_kernel.cu:391-458, schema ps_roi_align.cpp:76-77).
 * grad [num_rois, C_out, pooled_h, pooled_w] DENSE (the shim makes it contiguous), rois [num_rois, 5],
 * grad_input [batch, channels, height, width] - written IN FULL (no pre-zeroing).  Unlike the reference (atomics,
 * alertNotDeterministic), with `deterministic` != 0 (the shim passes torch.are_deterministic_algorithms_enabled(); the
 * reference raises in that mode) all four backward ops are bit-reproducible for F32, F64 and F16, every sampling_ratio
 * (adaptive included) and any plane size: grad_input is accumulated in shared memory (fp32; fp64 for F64) one row tile of
 * one plane at a time, by row-owning warps in a fixed order that does not depend on the tiling, and rounded once to the
 * storage type.  Two cases still run the atomic scatter with `deterministic` != 0: a grad_input row that does not fit in
 * shared memory (vb200_roi_backward_deterministic_supported() == 0; about 58 000 fp32 / 29 000 fp64 columns on an H100),
 * and a workspace that is missing or smaller than vb200_roi_backward_workspace_bytes().  With `deterministic` == 0 nothing
 * changed: roi_align fp32 with sampling_ratio 1..8 on a plane that fits accumulates plane by plane in shared memory - with
 * shared-memory atomics and the RoIs dealt round-robin to the warps for tables of at most 32 y samples, 32 x taps and 64
 * bins, with the row-owning kernel above that - and everything else scatters with global atomics.
 * workspace: vb200_roi_backward_workspace_bytes() bytes (row headers and sampling tables, the same for every dtype; pass
 * sampling_ratio 1 for roi_pool and ps_roi_pool). */
VB200_API size_t vb200_roi_backward_workspace_bytes(int num_rois, int pooled_h, int pooled_w, int sampling_ratio);
/* 1 when the deterministic backward of the RoI ops takes a grad_input of this dtype, height and width on the current
 * device (one row must fit in shared memory), 0 when it would fall back to the atomic scatter. */
VB200_API int vb200_roi_backward_deterministic_supported(int dtype, int height, int width);
VB200_API int vb200_roi_align_backward(const void* grad, const void* rois, void* grad_input, int dtype, int batch,
                             int channels, int height, int width, int num_rois, int pooled_h, int pooled_w,
                             double spatial_scale, int sampling_ratio, int aligned, int deterministic,
                             void* workspace, size_t workspace_bytes, vb200_stream stream);
VB200_API int vb200_roi_pool_backward(const void* grad, const void* rois, const int32_t* argmax, void* grad_input, int dtype,
                            int batch, int channels, int height, int width, int num_rois, int pooled_h, int pooled_w,
                            double spatial_scale, int deterministic, void* workspace, size_t workspace_bytes,
                            vb200_stream stream);
VB200_API int vb200_ps_roi_align_backward(const void* grad, const void* rois, const int32_t* channel_mapping, void* grad_input,
                                int dtype, int batch, int channels, int height, int width, int num_rois, int pooled_h,
                                int pooled_w, double spatial_scale, int sampling_ratio, int deterministic,
                                void* workspace, size_t workspace_bytes, vb200_stream stream);

/* ---- nms ---------------------------------------------------------------
 * Replaces nms_kernel, csrc/ops/cuda/nms_kernel.cu:166-258 (schema
 * torchvision::nms, csrc/ops/nms.cpp:27).  boxes [n,4] (x1,y1,x2,y2), scores [n].
 * Writes the kept ORIGINAL indices, in descending-score order (stable), to
 * keep_out[0..*num_keep_out) — both device memory, keep_out sized n.  The
 * caller reads *num_keep_out (the reference's masked_select sync).
 * dtype: F32, F64 or F16 - the three instantiations of the reference kernel, each with the arithmetic of its compiled
 * reference (F16: devIoU<Half> mixes half and float roundings, nms_kernel.cu:42-54; VB200_NMS_CUDA only).
 * workspace: sort buffers + the n x ceil(n/64) 64-bit IoU matrix (about n*n/8 bytes: 1.2 MB at
 * n = 3 000, 50 MB at 20 000, 1.25 GB at 100 000 - the reference allocates the same matrix). */
VB200_API size_t vb200_nms_workspace_bytes(int64_t n);
VB200_API int vb200_nms(const void* boxes, const void* scores, int dtype, int64_t n, double iou_threshold,
              int semantics, void* workspace, size_t workspace_bytes, int64_t* keep_out,
              int64_t* num_keep_out, vb200_stream stream);

/* ---- batched_nms -------------------------------------------------------
 * Replaces the Python torchvision.ops.boxes.batched_nms (boxes.py:57-126):
 * one fused device pipeline instead of a per-class Python loop.  idxs [n] int64.
 * Output as vb200_nms (or *num_keep_out = -1, see VB200_BNMS_WIDE_KEYS).  strategy: VB200_BNMS_*.
 * workspace: sort buffers + 33 mask words per box (42 MB at n = 100 000); the plain-nms matrix is
 * included only up to the reference's coordinate-trick range (4 n <= 100 000) - VB200_BNMS_TRICK
 * forced on a larger problem runs the sequential per-segment kernel instead. */
VB200_API size_t vb200_batched_nms_workspace_bytes(int64_t n);
VB200_API int vb200_batched_nms(const void* boxes, const void* scores, const int64_t* idxs, int dtype,
                      int64_t n, double iou_threshold, int semantics, int strategy,
                      void* workspace, size_t workspace_bytes, int64_t* keep_out,
                      int64_t* num_keep_out, vb200_stream stream);

/* ---- detection post-processing around batched_nms -------------------------
 * Replaces the per-image tail of RoIHeads.postprocess_detections (torchvision/models/detection/roi_heads.py:700-737)
 * and RegionProposalNetwork.filter_proposals (rpn.py:273-298): clip_boxes_to_image -> score filter (`>` or `>=`) ->
 * remove_small_boxes -> batched_nms -> keep[:topk] -> gather boxes / scores / labels, as one device pipeline.
 * boxes [n,4] F32, scores [n] F32, labels [n] int64 (class ids / FPN level ids); outputs sized min(n, topk).
 * SYNCHRONOUS: the candidate count decides the reference's batched_nms strategy (boxes.py:86) and the output count sizes
 * the result, so the call synchronises `stream` twice and returns the number of detections in *count_host (host). */
VB200_API size_t vb200_detection_postprocess_workspace_bytes(int64_t n);
VB200_API int vb200_detection_postprocess(const void* boxes, const void* scores, const int64_t* labels, int dtype, int64_t n,
                                double img_h, double img_w, double score_thresh, int score_inclusive, double min_size,
                                double iou_threshold, int64_t topk, int semantics, void* workspace,
                                size_t workspace_bytes, void* boxes_out, void* scores_out, int64_t* labels_out,
                                int64_t* count_host, vb200_stream stream);

/* ---- single-stage detector post-processing --------------------------------------------------------------------
 * Replaces postprocess_detections of RetinaNet (torchvision/models/detection/retinanet.py:509-571), FCOS
 * (fcos.py:489-556) and SSD / SSDLite (ssd.py:414-463): per image, per FPN level (or per foreground class) score,
 * `score > score_thresh`, topk(topk_candidates), decode (BoxCoder.decode_single, _utils.py:183-224, or
 * BoxLinearCoder.decode, _utils.py:275-310) and clip_boxes_to_image of the selected items, then batched_nms ->
 * keep[:detections_per_img] -> gather, for every image of the call in one device pipeline.
 *   kind VB200_SS_RETINANET: score = sigmoid(logit), segment = (image, level) slice of [A_l, C] logits, flattened;
 *        VB200_SS_FCOS:      score = sqrt(sigmoid(logit) * sigmoid(ctrness)), BoxLinearCoder(normalize_by_size=True);
 *        VB200_SS_SSD:       score = the [A, C] softmax probabilities (num_levels = 1), segment = (image, class >= 1).
 * Within a segment the top min(topk_candidates, n_pass) items are ordered by score descending, then flat index
 * ascending; labels are flat index % C (RetinaNet, FCOS) or the class (SSD).
 * HOST arrays (one entry per level unless noted): level_anchors (A_l); logits / ctrness / regression device pointers
 * of [N, A_l, C] / [N, A_l, 1] / [N, A_l, 4] fp32 tensors whose last dimension is dense, with (image, row) strides in
 * elements; anchors: N * L device pointers (image-major) of [A_l, 4] fp32 with their row strides; image_hw: 2N sizes;
 * weights: the BoxCoder's 4 weights (ignored by FCOS).  topk_candidates <= VB200_SS_MAX_TOPK.
 * Output: boxes_out [N * detections_per_img, 4] / scores_out / labels_out (int64) receive the detections of every
 * image, concatenated; counts_host [N] (host) their per-image numbers.
 * SYNCHRONOUS: reads the candidate counts of all images (they decide each image's batched_nms strategy,
 * boxes.py:86) and then the kept counts of all images - two synchronisations of `stream` per call. */
enum { VB200_SS_RETINANET = 0, VB200_SS_FCOS = 1, VB200_SS_SSD = 2 };
#define VB200_SS_MAX_TOPK 2048
VB200_API size_t vb200_single_stage_postprocess_workspace_bytes(int kind, int num_images, int num_levels,
                                                      const int64_t* level_anchors, int num_classes,
                                                      int64_t topk_candidates, int64_t detections_per_img);
VB200_API int vb200_single_stage_postprocess(int kind, int num_images, int num_levels, const int64_t* level_anchors,
                                   int num_classes, const void* const* logits, const int64_t* logit_strides,
                                   const void* const* ctrness, const int64_t* ctrness_strides,
                                   const void* const* regression, const int64_t* regression_strides,
                                   const void* const* anchors, const int64_t* anchor_strides, const double* image_hw,
                                   double score_thresh, int64_t topk_candidates, double nms_thresh,
                                   int64_t detections_per_img, const double* weights, double bbox_xform_clip,
                                   int semantics, void* workspace, size_t workspace_bytes, void* boxes_out,
                                   void* scores_out, int64_t* labels_out, int64_t* counts_host, vb200_stream stream);

/* ---- Keypoint R-CNN keypoints from heatmaps ------------------------------------------------------------------------
 * Replaces heatmaps_to_keypoints, torchvision/models/detection/roi_heads.py:237-307 (its per-RoI loop of bicubic
 * F.interpolate, argmax and coordinate arithmetic), for all RoIs of a call at once.
 * maps [K, N, H, W] (F32 / F16 / BF16, H and W at most VB200_KP_MAX_SIDE), rois [K, 4] fp32 (x1, y1, x2, y2).
 * Per RoI the map is resized to ceil(max(y2 - y1, 1)) x ceil(max(x2 - x1, 1)) as ATen's CUDA upsample_bicubic2d does it
 * (align_corners=False, the result rounded to the map dtype, a same-size map copied unchanged), and each keypoint's argmax
 * (NaN above everything, ties and NaNs to the lowest index) is mapped back into the image with the reference's fp32
 * arithmetic.  Output: xy_out [K, 3, N] (x, y, then a row of ones; the reference returns its permute(0, 2, 1)) and
 * scores_out [K, N], the resized map's value at the argmax.  A box whose resized map has a non-finite size or 2^31 or more
 * pixels (the reference raises for the first and cannot allocate the second) gets NaN outputs.
 * workspace: vb200_heatmaps_to_keypoints_workspace_bytes(K, N) bytes, a function of the shapes only.  Three launches
 * whatever K; asynchronous. */
#define VB200_KP_MAX_SIDE 128
VB200_API size_t vb200_heatmaps_to_keypoints_workspace_bytes(int64_t num_rois, int num_keypoints);
VB200_API int vb200_heatmaps_to_keypoints(const void* maps, int dtype, const float* rois, int64_t num_rois, int num_keypoints,
                                          int height, int width, float* xy_out, float* scores_out, void* workspace,
                                          size_t workspace_bytes, vb200_stream stream);

/* ---- detection model input batching ---------------------------------------------------------------------------------
 * Replaces GeneralizedRCNNTransform.forward's inference loop, torchvision/models/detection/transform.py:119-158 with
 * normalize (:160-169), _resize_image_and_masks (:25-83) and batch_images (:237-255), for all images at once.
 * Image i is [channels, in_h, in_w] at `data` with element strides (stride_c, stride_h, stride_w), read in place.  Each
 * element of the padded batch output [num_images, channels, pad_h, pad_w] (contiguous, `dtype` = F32 / F16 / BF16 for
 * every image) is either +0.0 or pixel (y, x) of image i normalized and resized to out_h x out_w: (v - mean[c]) and then
 * / std[c], each computed in fp32 and rounded to the dtype, then ATen's CUDA upsample_bilinear2d (align_corners=False,
 * scale (float)in / out, fp32 blend; an image whose size does not change is copied, as ATen's kernel does) of those
 * values, rounded to the dtype.  mean_host / std_host: HOST arrays of
 * `channels` floats (<= 8 channels), already rounded to the dtype.  One launch per VB200_RCNN_MAX_IMAGES images. */
#define VB200_RCNN_MAX_IMAGES 256
typedef struct vb200_rcnn_image {
  const void* data;
  int64_t stride_c, stride_h, stride_w;
  int in_h, in_w, out_h, out_w;
} vb200_rcnn_image;
VB200_API int vb200_rcnn_batch_images(const vb200_rcnn_image* images, int num_images, int channels, int dtype, int pad_h,
                                      int pad_w, const float* mean_host, const float* std_host, void* output,
                                      vb200_stream stream);

/* ---- detection output rescaling ---------------------------------------------------------------------------------------
 * Replaces GeneralizedRCNNTransform.postprocess's resize_boxes and resize_keypoints, transform.py:257-277, 288-319, for
 * all images at once.  Item k is a fp32 [rows, cols, width] array (boxes: cols 1, width 4; keypoints: width 3) read with
 * in_stride and written with out_stride (elements): columns 0 and 2 of a box and column 0 of a keypoint are multiplied
 * by ratio_w, columns 1 and 3 of a box and column 1 of a keypoint by ratio_h (each a single fp32 product), a keypoint's
 * column 2 is copied.  ratio_w / ratio_h: the fp32 quotient new / original size.  One launch per VB200_RCNN_MAX_RESCALE
 * items. */
#define VB200_RCNN_MAX_RESCALE 128
typedef struct vb200_rcnn_rescale_item {
  const float* input;
  float* output;
  int64_t in_stride[3], out_stride[3];
  int64_t rows;
  int cols, width;
  float ratio_w, ratio_h;
} vb200_rcnn_rescale_item;
VB200_API int vb200_rcnn_rescale(const vb200_rcnn_rescale_item* items, int num_items, vb200_stream stream);

/* ---- training-target assignment (box matching) ------------------------------------------------------------------------
 * Replaces the per-image loops of RegionProposalNetwork.assign_targets_to_anchors (torchvision/models/detection/rpn.py:193-229),
 * RoIHeads.assign_targets_to_proposals (roi_heads.py:580-613) and the top of RetinaNet.compute_loss (retinanet.py:494-507):
 * box_iou(gt, predictions) (ops/boxes.py:308-370), Matcher.__call__ and set_low_quality_matches_ (_utils.py:357-416) and
 * the callers' masked writes, for all images of a call, without the M x N IoU matrix.
 * Image i: gt [num_gt, 4] of gt_dtype and predictions [num_pred, 4] of pred_dtype (x1, y1, x2, y2; element strides
 * (row, column)).  IoU follows box_iou op by op: fp32 for any mix of F32 / F16 / BF16 (rb - lt rounded to the dtype when
 * both sides are F16, or both BF16), fp64 when both are F64.  Each prediction's best gt is Tensor.max(dim=0)'s (ascending gt
 * order, ties to the lowest index, the first NaN wins); it becomes -1 below low_threshold and -2 in [low, high), compared
 * with the threshold rounded to float (double for F64); with allow_low_quality a prediction whose IoU equals some gt's max
 * over the image's predictions keeps its best gt.  Outputs, per mode (num_pred entries each, dense):
 *   VB200_MATCH_RAW        out0 int64 matches (all -1 when num_gt == 0)
 *   VB200_MATCH_RPN        out0 float labels (1 matched, 0 for -1, -1 for -2), out1 [num_pred, 4] of gt_dtype =
 *                          gt[max(match, 0)]; when num_gt == 0 both are fp32 zeros
 *   VB200_MATCH_ROI_HEADS  out0 int64 max(match, 0), out1 int64 gt_labels[max(match, 0)], 0 for -1, -1 for -2 (gt_labels
 *                          int64 with element stride label_stride); when num_gt == 0 both are zeros
 * An image with num_gt > 0 and num_pred == 0 is an error (the reference raises "No proposal boxes available").
 * workspace: vb200_match_boxes_workspace_bytes(total gt boxes of the call, VB200_F64 when both sides are F64 else
 * VB200_F32, allow_low_quality) bytes, a function of the shapes only (the per-gt max keys; 0 without allow_low_quality).
 * Per VB200_MATCH_MAX_IMAGES images: two kernel launches with allow_low_quality (the gt maxima, then the matches), one
 * without, plus one memset of the keys per call.  Asynchronous. */
#define VB200_MATCH_MAX_IMAGES 64
enum { VB200_MATCH_RAW = 0, VB200_MATCH_RPN = 1, VB200_MATCH_ROI_HEADS = 2 };
typedef struct vb200_match_image {
  const void* gt;
  const void* pred;
  const int64_t* gt_labels;
  void* out0;
  void* out1;
  int64_t gt_stride[2], pred_stride[2], label_stride;
  int64_t num_pred;
  int num_gt;
} vb200_match_image;
VB200_API size_t vb200_match_boxes_workspace_bytes(int64_t total_gt, int dtype, int allow_low_quality);
VB200_API int vb200_match_boxes(const vb200_match_image* images, int num_images, int gt_dtype, int pred_dtype, int mode,
                                double high_threshold, double low_threshold, int allow_low_quality, void* workspace,
                                size_t workspace_bytes, vb200_stream stream);

/* ---- FCOS training-target assignment (centre sampling) ------------------------------------------------------------------
 * Replaces the per-image matching loop of FCOS.compute_loss (torchvision/models/detection/fcos.py:440-487, the [N, M]
 * tensors of :455-483) for all images of a call, without any N x M intermediate.
 * Image i: gt [num_gt, 4] of gt_dtype and anchors [num_anchors, 4] of anchor_dtype (x1, y1, x2, y2; element strides
 * (row, column)); out int64 [num_anchors], dense.  Per anchor, op by op as the reference: centres, sizes, radius * size and
 * the level bounds size * 4 / size * 8 rounded to anchor_dtype, gt centres and areas rounded to gt_dtype, anchor - gt
 * differences rounded to the promoted type (the dtype when both sides share it, fp32 for any other mix of F32 / F16 / BF16,
 * fp64 when both are F64), scalars rounded to float unless both are F64; the strict comparisons with NaN failing them;
 * value = (float)match * (1e8 - area) in promote(fp32, gt_dtype); the best gt as Tensor.max(dim=1) picks it (ascending gt
 * order, ties to the lowest index, the first NaN wins), -1 where that value is below 1e-5.  An image with num_gt == 0 gets
 * all -1.  The lower bound is 0 for the first and the upper bound inf from the last anchors that
 * vb200_fcos_level_bounds(num_anchors, first_level, last_level) names, first_level / last_level being
 * num_anchors_per_level[0] / [-1].  One kernel launch per VB200_MATCH_MAX_IMAGES images, no workspace.  Asynchronous. */
typedef struct vb200_fcos_image {
  const void* gt;
  const void* anchors;
  int64_t* out;
  int64_t gt_stride[2], anchor_stride[2];
  int64_t num_anchors;
  int num_gt;
} vb200_fcos_image;
/* Python's slicing of lower_bound[:first_level] = 0 and upper_bound[-last_level:] = inf (fcos.py:472-475) over num_anchors
 * anchors: *lower_end_host anchors from the front get lower bound 0, anchors from *upper_begin_host on get upper bound inf
 * (a last_level of 0 makes [-0:] the whole tensor; counts beyond num_anchors clamp; negative counts index from the end). */
VB200_API void vb200_fcos_level_bounds(int64_t num_anchors, int64_t first_level, int64_t last_level, int64_t* lower_end_host,
                                       int64_t* upper_begin_host);
VB200_API int vb200_fcos_match(const vb200_fcos_image* images, int num_images, int gt_dtype, int anchor_dtype, double radius,
                               int64_t first_level, int64_t last_level, vb200_stream stream);

/* ---- single-stage detector head losses ----------------------------------------------------------------------------------
 * Replace, forward and backward, for all images of a call with no host sync and no full-size intermediate:
 *   VB200_LOSS_RETINANET_CLS  the per-image loop of RetinaNetClassificationHead.compute_loss
 *                             (torchvision/models/detection/retinanet.py:158-189, with sigmoid_focal_loss, ops/focal_loss.py:41-56,
 *                             alpha 0.25, gamma 2);
 *   VB200_LOSS_RETINANET_BOX  that of RetinaNetRegressionHead.compute_loss (retinanet.py:272-302 with _box_loss "l1",
 *                             models/detection/_utils.py:524-526, and encode_boxes, :103-118);
 *   VB200_LOSS_FCOS_CLS, _BOX FCOSHead.compute_loss (fcos.py:52-125): its per-image gather loop, the .item() host sync,
 *                             sigmoid_focal_loss (alpha 0.25, gamma 2), BoxLinearCoder.decode / .encode (_utils.py:240-310),
 *                             generalized_box_iou_loss (ops/giou_loss.py with _loss_inter_union, ops/_utils.py:87-105) and
 *                             binary_cross_entropy_with_logits on the centre-ness; the classification loss in one call, the GIoU
 *                             and centre-ness losses together in the other.
 * Image i, all fp32: pred is the image's dense rows of cls_logits [A, C] or bbox_regression [A, 4] (unit stride, rows of
 * `width` = C for the classification kinds, 4 for the box kinds); matched int64 [A] (element stride matched_stride); labels
 * int64 [num_gt] (stride label_stride; not RETINANET_BOX); gt [num_gt, 4] and anchors [A, 4] (element strides (row, column);
 * box kinds only); ctrness the image's bbox_ctrness [A] (element stride ctrness_stride, FCOS_BOX only); grad / grad_ctrness
 * (backward only; grad_ctrness FCOS_BOX only) the image's dense rows of the gradients, written exactly once.  A call ignores
 * the fields its kind does not use.  A bad index (per kind below) makes the loss NaN and the anchor's gradient rows NaN
 * where the reference raises a device-side assert; nothing outside labels, gt or the pred rows is read.
 * Arguments: weights_host (RETINANET_BOX only, required) the box coder's weights as torch.as_tensor(weights, dtype=float32)
 * rounds them; normalize_by_size (read for FCOS_BOX only) the BoxLinearCoder's flag (nonzero: the codes are relative to the
 * anchor's width and height); loss / loss2 (device fp32, 0-dim) the losses, loss2 required for FCOS_BOX and null otherwise;
 * grad_loss / grad_loss2 (device fp32, 0-dim) their incoming gradients, grad_loss2 for FCOS_BOX only, not both null.
 * Every sum is in a fixed order, no floating-point atomics: results are bit-reproducible.  workspace: the query's bytes, a
 * function of (kind, B, A) only.  Per VB200_LOSS_MAX_IMAGES images one kernel launch, plus one finalize launch per forward.
 * A * width must be below 2^31.  An unknown kind is VB200_EINVAL.  Asynchronous.
 *
 * RetinaNet.  matched holds the Matcher's indices: >= 0 foreground, -2 ignored, other negatives background; the target class
 * of a foreground anchor is labels[matched], a label in [-C, 0) wrapping as indexing does.  A matched index >= num_gt or a
 * label outside [-C, C) is bad: the image's loss is NaN and its gradient rows NaN.  Forward: *loss = (sum_i L_i) * fl(1 / B)
 * with the images added in order, L_i = S_i / max(1, n_i) as the heads divide (a true division in the classification head,
 * the product with fl(1 / n_i) in the regression head), S_i the image's sum, n_i its foreground count (written to
 * num_foreground[i], device int64).  Classification elements follow the focal loss in stable fp32 forms, the regression
 * targets are encode_single's bits.  Backward: grad_loss times the per-image scale fl(fl(g * fl(1 / B)) / max(1, n_i)) (the
 * product with fl(1 / n_i) for regression) times the element's derivative; 0 for ignored and background-regression rows,
 * sign(pred - target) as torch.sign (0 for ±0 and NaN).
 *
 * FCOS.  Foreground, as the reference derives it with m = matched[a]: m < 0 (-2 included) is background; an image with no gt
 * and m >= 0 has target class 0 and the zero gt box; otherwise l = labels[m] is the target class if l >= 0 and background if
 * l < 0 (not wrapped).  m >= num_gt > 0, or (classification) l >= C, is bad: the loss is NaN and the anchor's gradient rows
 * NaN.  n = the number of foreground anchors of the whole batch (bad ones included), written to *num_foreground (device
 * int64).  Forward: each of *loss, *loss2 = fl(S) * fl(1 / max(1, n)), S the sum over the whole batch (the head divides by
 * the Python int from .item(), which ATen's CUDA division turns into the product with its fp32 reciprocal; no 1 / B).
 * Classification: the focal loss of every element, in the stable forms of the RetinaNet kind.  Box: per foreground anchor
 * the GIoU loss of decode(bbox_regression, anchor) against the gt box (*loss), and BCE-with-logits (1 - t) x - log sigmoid(x)
 * of the centre-ness logit x against t = sqrt(min(l, r) / max(l, r) * min(t, b) / max(t, b)) of encode(anchor, gt) (*loss2);
 * decode, encode and the GIoU restated op by op in fp32, so every branch (overlap, min / max) is the reference's fp32
 * decision.  Backward: s = fl(g * fl(1 / max(1, n))), g read from device memory, times each element's derivative; the GIoU
 * gradient is analytic through the decode, with torch.max / torch.min's tie rule (equal operands get half the gradient
 * each), and the centre-ness gradient s (sigmoid(x) - t).  Non-foreground rows are exactly 0; a null grad_loss or grad_loss2
 * counts as a zero gradient: its rows are 0. */
#define VB200_LOSS_MAX_IMAGES 64
enum { VB200_LOSS_RETINANET_CLS, VB200_LOSS_RETINANET_BOX, VB200_LOSS_FCOS_CLS, VB200_LOSS_FCOS_BOX };
typedef struct vb200_loss_image {
  const float* pred;
  const float* ctrness;        /* FCOS box only */
  const int64_t* matched;
  const int64_t* labels;       /* not RetinaNet box */
  const float* gt;             /* box kinds only */
  const float* anchors;        /* box kinds only */
  float* grad;                 /* backward only */
  float* grad_ctrness;         /* FCOS box backward only */
  int64_t ctrness_stride, matched_stride, label_stride, gt_stride[2], anchor_stride[2];
  int64_t num_gt;
} vb200_loss_image;
VB200_API size_t vb200_head_loss_workspace_bytes(int kind, int num_images, int64_t num_anchors);
VB200_API int vb200_head_loss(int kind, const vb200_loss_image* images, int num_images, int64_t num_anchors, int width,
                              const float* weights_host, int normalize_by_size, float* loss, float* loss2, int64_t* num_foreground,
                              void* workspace, size_t workspace_bytes, vb200_stream stream);
VB200_API int vb200_head_loss_backward(int kind, const vb200_loss_image* images, int num_images, int64_t num_anchors, int width,
                                       const float* weights_host, int normalize_by_size, const float* grad_loss,
                                       const float* grad_loss2, const int64_t* num_foreground, vb200_stream stream);

/* ---- Mask R-CNN mask loss ------------------------------------------------------------------------------------------------
 * Replaces, forward and backward, for all images of a call, maskrcnn_loss (torchvision/models/detection/roi_heads.py:100-129)
 * with project_masks_on_boxes (:85-97): the fp32 copy of every image's whole gt-mask stack, roi_align over it, the label
 * gather, the two torch.cat, the [P, C, M, M] advanced-index gather, binary_cross_entropy_with_logits as a chain of
 * elementwise kernels and a mean, and in the backward the zeros_like + index_put of the dense gradient.
 * Image i: masks its gt masks [num_gt, height, width] (element strides mask_stride; mask_dtype VB200_U8, bool masks passed
 * as their 0 / 1 bytes with VB200_U8), read in place, never copied; proposals its positive RoIs fp32 [num_rois, 4] (x1, y1,
 * x2, y2; element strides (row, column)); matched int64 [num_rois] (stride matched_stride), the gt index of each RoI; labels
 * int64 [num_gt] (stride label_stride).  The images' RoIs are the rows of mask_logits in order: mask_logits fp32 [P, C, M, M]
 * dense, P = sum of num_rois, C = num_classes, M = size; targets fp32 [P, M, M] dense; P * C * M * M below 2^31.
 * Arithmetic: RoI p of image i with m = matched[p] has target t[p, bin] = roi_align(float(masks[m]), proposals[p], (M, M),
 * spatial_scale 1, sampling_ratio -1, aligned false) -- the reference's RoI geometry, sample order and roundings, bit-exact
 * with its CPU kernel -- and logit x = mask_logits[p, l, bin] with l = labels[m], a label in [-C, 0) wrapping as indexing
 * does.  Each element's BCE term (1 - t) x + softplus(-x) is formed in fp64 from fp32 exp / log1p (the stable forms of the
 * head losses).  Forward: *loss = fl(S) * fl(1 / N), N = P * M * M (ATen's mean: the sum, then the product with the fp32
 * reciprocal), S the sum of every term: per CTA of 256 (RoI, bin) threads a fixed-order tree, the CTA partials added in
 * order by one finalize CTA.  targets are written (the backward reads them).  Backward: grad_logits [P, C, M, M] dense,
 * written exactly once: the label plane of RoI p gets fl(s * (sigmoid(x) - t)) with s = fl(g * fl(1 / N)), g = *grad_loss
 * read from device memory; every other plane +0; a null grad_loss is a zero gradient (every element +0).
 * Bad indices, where the reference raises a device-side assert: m < 0, m >= num_gt or a label outside [-C, C) makes the loss
 * NaN, the RoI's targets NaN and its whole [C, M, M] gradient block NaN; nothing outside masks, labels, proposals, matched
 * and the RoI's logits is read.  No floating-point atomics and nothing from the SM count: bit-reproducible in every mode.
 * Launches: per VB200_LOSS_MAX_IMAGES images one forward kernel (none for images without RoIs) plus one finalize per forward;
 * one backward kernel per VB200_LOSS_MAX_IMAGES images.  workspace: the query's bytes, a function of (num_images, P, M) only.
 * P = 0 writes NaN (0 / 0) and launches only the finalize.  Asynchronous. */
typedef struct vb200_mask_image {
  const void* masks;
  const float* proposals;
  const int64_t* matched;
  const int64_t* labels;
  int64_t mask_stride[3], proposal_stride[2], matched_stride, label_stride;
  int64_t num_gt, height, width, num_rois;
  int mask_dtype;
} vb200_mask_image;
VB200_API size_t vb200_mask_loss_workspace_bytes(int num_images, int64_t total_rois, int size);
VB200_API int vb200_mask_loss(const vb200_mask_image* images, int num_images, const float* mask_logits, int num_classes, int size,
                              float* loss, float* targets, void* workspace, size_t workspace_bytes, vb200_stream stream);
VB200_API int vb200_mask_loss_backward(const vb200_mask_image* images, int num_images, const float* mask_logits, const float* targets,
                                       int num_classes, int size, const float* grad_loss, float* grad_logits, vb200_stream stream);

/* ---- deform_conv2d -----------------------------------------------------
 * Replaces deform_conv2d_forward_kernel, csrc/ops/cuda/deform_conv2d_kernel.cu:1035-1255
 * (schema torchvision::deform_conv2d, csrc/ops/deform_conv2d.cpp:101-102).
 * input [batch,c_in,in_h,in_w], weight [c_out,c_in/groups,kh,kw],
 * offset [batch, offset_groups*2*kh*kw, out_h, out_w],
 * mask [batch, offset_groups*kh*kw, out_h, out_w] (ignored if !use_mask),
 * bias [c_out] (may be NULL), out [batch,c_out,out_h,out_w].
 * dtype: BF16 / F16 (wgmma tensor-core path, fp32 accumulate), F32 (wgmma with a three-way bf16 split of both
 * operands, six MMAs per K step: fp32-level accuracy; SIMT kernel for shapes the tensor-core tiling does not cover),
 * F64 (plain double kernel - the reference's gradcheck tests run in double).
 * workspace: vb200_deform_conv2d_workspace_bytes() bytes (may be 0). */
VB200_API size_t vb200_deform_conv2d_workspace_bytes(int dtype, int batch, int c_in, int in_h, int in_w,
                                           int c_out, int kh, int kw, int out_h, int out_w,
                                           int groups, int offset_groups);

/* Weights are constant across inference calls and a channels-last producer can hand the input over without the
 * NCHW -> NHWC staging pass: vb200_deform_conv2d_pack_weight() writes the swizzled K-major image the tensor-core
 * kernels read (vb200_deform_conv2d_packed_weight_bytes() bytes; 0 = this shape takes the SIMT kernel), and
 * vb200_deform_conv2d_forward() takes it (packed_weight may be NULL) plus `input_is_nhwc` (input laid out
 * [batch, in_h, in_w, c_in], 16-byte aligned).  The torch shim caches the packed image per weight tensor / version. */
VB200_API size_t vb200_deform_conv2d_packed_weight_bytes(int dtype, int c_in, int c_out, int kh, int kw, int groups, int offset_groups);
VB200_API int vb200_deform_conv2d_pack_weight(const void* weight, void* packed, int dtype, int c_in, int c_out, int kh, int kw,
                                    int groups, int offset_groups, vb200_stream stream);
/* outs[0] is the output; outs[1..n_outs) (1 <= n_outs <= 8) fuse the all-gather of the output over the GPUs of one box
 * (SURVEY.md 8e: the batch shards, one all-gather of the per-shard outputs): outs[0] is then the caller's slot of its own
 * gathered buffer and outs[1..n_outs) the SAME slot of every peer's buffer (peer-mapped device pointers); the wgmma kernel's
 * epilogue stores each output element to all of them.  The caller synchronises the ranks before anyone reads.  n_outs = 1
 * is the plain op. */
VB200_API int vb200_deform_conv2d_forward(const void* input, const void* weight, const void* packed_weight, int input_is_nhwc,
                                const void* offset, const void* mask, const void* bias, void* const* outs, int n_outs,
                                int dtype, int batch, int c_in, int in_h, int in_w, int c_out, int kh, int kw,
                                int stride_h, int stride_w, int pad_h, int pad_w, int dil_h, int dil_w, int groups,
                                int offset_groups, int use_mask, void* workspace, size_t workspace_bytes,
                                vb200_stream stream);

/* ---- deform_conv2d backward ----------------------------------------------
 * Replace the kernels of deform_conv2d_backward_kernel, csrc/ops/cuda/deform_conv2d_kernel.cu:319-1033 (schema
 * csrc/ops/deform_conv2d.cpp:103-104).  The two dense contractions (weight^T x grad_out, grad_out x columns^T) are plain
 * GEMMs issued by the caller (the torch shim uses cuBLAS through at::matmul); these entry points are the passes around them:
 *   vb200_deform_conv2d_sample_columns: columns [n_imgs, c_in*kh*kw, out_h*out_w] = mask * bilinear(input) (replaces
 *     deformable_im2col, :136-209; layout is image-major here);
 *   vb200_deform_conv2d_backward_inputs: from dcol [n_imgs, c_in*kh*kw, out_h*out_w] = weight^T x grad_out, ONE pass writes
 *     grad_offset and grad_mask (no atomics) and scatters grad_input (atomics into a pre-zeroed tensor) - the reference's
 *     deformable_col2im_kernel (:319-401) and deformable_col2im_coord_kernel (:538-643) fused.
 * dtype: F32, F64, F16, BF16.  Weight groups are the caller's concern (c_in = all input channels). */
VB200_API int vb200_deform_conv2d_sample_columns(const void* input, const void* offset, const void* mask, void* columns, int dtype,
                                       int n_imgs, int c_in, int in_h, int in_w, int kh, int kw, int stride_h, int stride_w,
                                       int pad_h, int pad_w, int dil_h, int dil_w, int offset_groups, int use_mask,
                                       vb200_stream stream);
/* Bit-reproducible grad_input (the reference instead raises under torch.use_deterministic_algorithms,
 * alertNotDeterministic("compute_grad_input"), deformable_col2im's caller :441).  With `deterministic` set,
 * vb200_deform_conv2d_backward_inputs writes grad_input IN FULL (no pre-zeroing) by a gather instead of the scatter: the
 * samples are binned by the cell (floor y, floor x) they fall in and sorted stably, and each grad_input[b, c, y, x] is summed
 * over the cells (y, x), (y, x-1), (y-1, x), (y-1, x-1) in that order, inside a cell in ascending (offset group, tap, output
 * pixel) order, in fp32 (double for F64) and rounded once.  The value depends on image b's data alone.  grad_offset /
 * grad_mask are the same as without the flag.  The workspace (vb200_deform_conv2d_backward_inputs_workspace_bytes, host
 * arithmetic only, 0 for an empty shape) holds the sort keys, the cell table and one record per sample; images are processed
 * in passes whose sample count fits int32 and key range fits 32 bits, and a shape whose single image exceeds that returns
 * VB200_EUNSUPPORTED before anything is launched.  With deterministic == 0 the workspace is unused and grad_input is
 * pre-zeroed and scattered with atomics, as described above. */
VB200_API size_t vb200_deform_conv2d_backward_inputs_workspace_bytes(int dtype, int n_imgs, int c_in, int in_h, int in_w, int kh, int kw,
                                                           int stride_h, int stride_w, int pad_h, int pad_w, int dil_h, int dil_w,
                                                           int offset_groups);
VB200_API int vb200_deform_conv2d_backward_inputs(const void* dcol, const void* input, const void* offset, const void* mask,
                                        void* grad_input, void* grad_offset, void* grad_mask, int dtype, int n_imgs, int c_in,
                                        int in_h, int in_w, int kh, int kw, int stride_h, int stride_w, int pad_h, int pad_w,
                                        int dil_h, int dil_w, int offset_groups, int use_mask, int deterministic,
                                        void* workspace, size_t workspace_bytes, vb200_stream stream);

/* ---- resize ------------------------------------------------------------
 * Replaces the interpolate path of resize_image,
 * torchvision/transforms/v2/functional/_geometry.py:340-360 (cast to fp32 ->
 * aten::upsample_bi{linear,cubic}2d[_aa] -> cast back) with ONE fused kernel:
 * reads `dtype`, computes in fp32, writes `dtype` (round-to-nearest-even for
 * floats; clamp(0,255)+round for U8 as _geometry.py:352-359).
 * input [planes, in_h, in_w] -> output [planes, out_h, out_w]; mode VB200_RESIZE_*;
 * align_corners=False semantics.  dtype: F32, F16, BF16, U8. */
VB200_API int vb200_resize(const void* input, void* output, int dtype, int64_t planes, int in_h, int in_w,
                 int out_h, int out_w, int mode, int antialias, vb200_stream stream);
/* resize fused with the all-gather of its output (SURVEY.md 8e: the batch shards over the GPUs of one box and the only
 * exchange is an all-gather of the per-shard outputs - here done by the kernel's own stores).  outputs[0] is the caller's
 * slot of its gathered buffer, outputs[1..n) the SAME slot of every peer's buffer (peer-mapped device pointers, e.g. from
 * torch.distributed._symmetric_memory or cudaIpcOpenMemHandle); each finished pixel is stored to all of them.  The caller
 * synchronises the ranks before peers read (and before the buffers are rewritten).  1 <= n_outputs <= 8.  Replaces the
 * `dist.all_gather` a data-parallel caller of resize_image (_geometry.py:283-362) issues after the op. */
VB200_API int vb200_resize_gather(const void* input, void* const* outputs, int n_outputs, int dtype, int64_t planes, int in_h,
                        int in_w, int out_h, int out_w, int mode, int antialias, vb200_stream stream);

/* ---- box_iou_rotated (API completeness, SURVEY.md §8f4) ------------------
 * Replaces box_iou_rotated_cuda, csrc/ops/cuda/box_iou_rotated_kernel.cu:92-160 (schema torchvision::box_iou_rotated,
 * csrc/ops/box_iou_rotated.cpp).  boxes1 [n1, 5], boxes2 [n2, 5] as (x_ctr, y_ctr, w, h, angle in degrees), F32;
 * ious [n1, n2] F32.  The intersection area is found by clipping (Sutherland-Hodgman) instead of the reference's
 * intersection points + convex hull: same area up to fp32 rounding. */
VB200_API int vb200_box_iou_rotated(const void* boxes1, const void* boxes2, float* ious, int dtype, int64_t n1, int64_t n2,
                          vb200_stream stream);

/* ---- fused inference preprocessing --------------------------------------
 * Replaces ImageClassification.forward, torchvision/transforms/_presets.py:57-64 (resize -> center_crop ->
 * convert_image_dtype(float) -> normalize) with one launch: only the crop window [crop_top, +crop_h) x [crop_left, +crop_w)
 * of the virtual resized image (resize_h x resize_w) is computed; the value is rounded to the storage dtype where the
 * reference materialises the resized image, scaled to [0, 1] for U8, then (x - mean[c]) / std[c].
 * input [batch, channels, in_h, in_w] (F32 / F16 / BF16 / U8), output [batch, channels, crop_h, crop_w] F32;
 * mean_host / std_host: HOST arrays of `channels` floats (<= 8 channels). */
VB200_API int vb200_resize_crop_normalize(const void* input, float* output, int dtype, int64_t batch, int channels, int in_h,
                                int in_w, int resize_h, int resize_w, int crop_top, int crop_left, int crop_h, int crop_w,
                                int mode, int antialias, const float* mean_host, const float* std_host, vb200_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* VISION_B200_H_ */
