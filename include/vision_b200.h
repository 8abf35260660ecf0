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

#define VB200_ABI_VERSION 1

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
/* Generation counter of those overrides (bumped by every (re)load): callers that cache work recorded under one setting
 * of them, e.g. captured CUDA graphs (as the library's own batched_nms graph cache does), key the cache on it. */
VB200_API int vb200_env_generation(void);

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
 * (schemas csrc/ops/ps_roi_pool.cpp:71-73).  Shapes as ps_roi_align; the backward zero-fills grad_input itself. */
VB200_API int vb200_ps_roi_pool_forward(const void* input, const void* rois, void* output, int32_t* channel_mapping, int dtype,
                              int batch, int channels, int height, int width, int num_rois, int pooled_h, int pooled_w,
                              double spatial_scale, vb200_stream stream);
VB200_API int vb200_ps_roi_pool_backward(const void* grad, const void* rois, void* grad_input, int dtype, int batch, int channels,
                               int height, int width, int num_rois, int pooled_h, int pooled_w, double spatial_scale,
                               vb200_stream stream);

/* ---- backward of the RoI ops --------------------------------------------
 * Replace roi_align_backward_kernel (csrc/ops/cuda/roi_align_kernel.cu:396-468, schema roi_align.cpp:76-77),
 * roi_pool_backward_kernel (cuda/roi_pool_kernel.cu:190-260, schema roi_pool.cpp:69-70) and
 * ps_roi_align_backward_kernel (cuda/ps_roi_align_kernel.cu:391-458, schema ps_roi_align.cpp:76-77).
 * grad [num_rois, C_out, pooled_h, pooled_w] DENSE (the shim makes it contiguous), rois [num_rois, 5],
 * grad_input [batch, channels, height, width] - written IN FULL (no pre-zeroing).  Unlike the reference (atomics,
 * alertNotDeterministic) the fp32 / fixed-sampling-grid path is bit-reproducible: every grad_input plane is
 * accumulated in shared memory by row-owning warps in a fixed order.  That path runs when `deterministic` != 0 (the shim
 * passes torch.are_deterministic_algorithms_enabled(); the reference raises in that mode), and for roi_align also when its
 * tables exceed 32 y samples, 32 x taps or 64 bins.  Otherwise, with `deterministic` == 0,
 * roi_align still accumulates plane by plane in shared memory, but with shared-memory atomics and the RoIs dealt
 * round-robin to the warps (no repeated work; summation order varies like the reference's), and roi_pool /
 * ps_roi_align - one bin per (RoI, plane) - scatter with global atomics.  Other dtypes (F16, F64),
 * adaptive sampling (sampling_ratio <= 0) and planes larger than shared memory use an atomic scatter kernel.
 * workspace: vb200_roi_backward_workspace_bytes() bytes (sampling tables; pass sampling_ratio 1 for roi_pool). */
VB200_API size_t vb200_roi_backward_workspace_bytes(int num_rois, int pooled_h, int pooled_w, int sampling_ratio);
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
VB200_API int vb200_deform_conv2d_forward(const void* input, const void* weight, const void* offset,
                                const void* mask, const void* bias, void* out, int dtype,
                                int batch, int c_in, int in_h, int in_w, int c_out, int kh,
                                int kw, int stride_h, int stride_w, int pad_h, int pad_w,
                                int dil_h, int dil_w, int groups, int offset_groups,
                                int use_mask, void* workspace, size_t workspace_bytes,
                                vb200_stream stream);

/* Weights are constant across inference calls and a channels-last producer can hand the input over without the
 * NCHW -> NHWC staging pass: vb200_deform_conv2d_pack_weight() writes the swizzled K-major image the tensor-core
 * kernels read (vb200_deform_conv2d_packed_weight_bytes() bytes; 0 = this shape takes the SIMT kernel), and
 * vb200_deform_conv2d_forward_ex() takes it (packed_weight may be NULL) plus `input_is_nhwc` (input laid out
 * [batch, in_h, in_w, c_in], 16-byte aligned).  The torch shim caches the packed image per weight tensor / version. */
VB200_API size_t vb200_deform_conv2d_packed_weight_bytes(int dtype, int c_in, int c_out, int kh, int kw, int groups, int offset_groups);
VB200_API int vb200_deform_conv2d_pack_weight(const void* weight, void* packed, int dtype, int c_in, int c_out, int kh, int kw,
                                    int groups, int offset_groups, vb200_stream stream);
VB200_API int vb200_deform_conv2d_forward_ex(const void* input, const void* weight, const void* packed_weight, int input_is_nhwc,
                                   const void* offset, const void* mask, const void* bias, void* out, int dtype, int batch,
                                   int c_in, int in_h, int in_w, int c_out, int kh, int kw, int stride_h, int stride_w,
                                   int pad_h, int pad_w, int dil_h, int dil_w, int groups, int offset_groups, int use_mask,
                                   void* workspace, size_t workspace_bytes, vb200_stream stream);
/* deform_conv2d fused with the all-gather of its output over the GPUs of one box (SURVEY.md 8e: the batch shards, one
 * all-gather of the per-shard outputs): outs[0] is the caller's slot of its own gathered buffer, outs[1..n_outs) the SAME slot
 * of every peer's buffer (peer-mapped device pointers); the wgmma kernel's epilogue stores each output element to all of
 * them.  Other arguments as vb200_deform_conv2d_forward_ex.  The caller synchronises the ranks before anyone reads. */
VB200_API int vb200_deform_conv2d_forward_gather(const void* input, const void* weight, const void* packed_weight, int input_is_nhwc,
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
VB200_API int vb200_deform_conv2d_backward_inputs(const void* dcol, const void* input, const void* offset, const void* mask,
                                        void* grad_input, void* grad_offset, void* grad_mask, int dtype, int n_imgs, int c_in,
                                        int in_h, int in_w, int kh, int kw, int stride_h, int stride_w, int pad_h, int pad_w,
                                        int dil_h, int dil_w, int offset_groups, int use_mask, vb200_stream stream);

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
