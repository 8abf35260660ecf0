"""Detection post-processing fused around batched_nms (SURVEY.md §8f3): drop-in bodies for
``RoIHeads.postprocess_detections`` (torchvision/models/detection/roi_heads.py:680-737) and
``RegionProposalNetwork.filter_proposals`` (rpn.py:242-298).  Everything up to the per-image loop (box decoding, softmax,
per-level top-k, sigmoid) is the reference's own tensor code; the per-image tail - clip, score filter, remove_small_boxes,
batched_nms, top-k, gathers - is ONE call of ``vision_b200::detection_postprocess`` per image.

The single-stage detectors' ``postprocess_detections`` (RetinaNet retinanet.py:509-571, FCOS fcos.py:489-556, SSD / SSDLite
ssd.py:414-463) are ONE call of ``vision_b200::single_stage_postprocess`` for all images: score, threshold, per-level (or
per-class) top-k, decode, clip, batched_nms and the top detections.  SSD keeps its softmax prologue as torch code.

Keypoint R-CNN's ``keypointrcnn_inference`` / ``heatmaps_to_keypoints`` (roi_heads.py:237-354), a per-detection loop of
bicubic resize, argmax and coordinate arithmetic, are ONE call of ``vision_b200::heatmaps_to_keypoints`` for all images.

``GeneralizedRCNNTransform.forward`` (transform.py:119-158), which every detection model enters through, is ONE call of
``vision_b200::rcnn_batch_images`` (normalize, bilinear resize and zero padding of all images); its ``postprocess``
(:257-277) rescales every image's boxes and keypoints with ONE call of ``vision_b200::rcnn_rescale``.

The training targets of ``RegionProposalNetwork.assign_targets_to_anchors`` (rpn.py:193-229),
``RoIHeads.assign_targets_to_proposals`` (roi_heads.py:580-613) and the matching loop of ``RetinaNet.compute_loss``
(retinanet.py:494-507), a per-image box_iou + Matcher, are ONE call of ``vision_b200::match_boxes`` for all images; the
centre-sampling matching loop of ``FCOS.compute_loss`` (fcos.py:440-487) is ONE call of ``vision_b200::fcos_match``.

RetinaNet's head losses, ``RetinaNetClassificationHead.compute_loss`` (retinanet.py:158-189, the sigmoid focal loss) and
``RetinaNetRegressionHead.compute_loss`` (:272-302, the "l1" box loss), per-image loops of full-size masks, gathers and
elementwise chains, are ONE call each of ``vision_b200::retinanet_cls_loss`` / ``retinanet_box_loss`` for all images, with
a fused backward (_autograd.py)."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F
from torch import Tensor

from . import _lib


# per-segment top-k capacity of the select kernel (VB200_SS_MAX_TOPK in include/vision_b200.h)
SINGLE_STAGE_MAX_TOPK = 2048
_SS_RETINANET, _SS_FCOS, _SS_SSD = 0, 1, 2


def _fusable(t: Tensor) -> bool:
    return isinstance(t, Tensor) and t.is_cuda and t.dtype == torch.float32 and not torch.jit.is_scripting() and not torch.jit.is_tracing()


def detection_postprocess(boxes: Tensor, scores: Tensor, labels: Tensor, image_shape, score_thresh: float, score_inclusive: bool,
                          min_size: float, nms_thresh: float, topk: int):
    """clip_boxes_to_image -> score filter -> remove_small_boxes -> batched_nms -> keep[:topk] -> (boxes, scores, labels)."""
    _lib.load_ops()
    h, w = image_shape
    return torch.ops.vision_b200.detection_postprocess(boxes, scores, labels, float(h), float(w), float(score_thresh),
                                                       bool(score_inclusive), float(min_size), float(nms_thresh), int(topk))


def roi_heads_postprocess_detections(self, class_logits, box_regression, proposals, image_shapes, _orig=None):
    """RoIHeads.postprocess_detections with the per-image tail fused (same outputs, same order)."""
    if not _fusable(class_logits):
        return _orig(self, class_logits, box_regression, proposals, image_shapes)
    device = class_logits.device
    num_classes = class_logits.shape[-1]
    boxes_per_image = [boxes_in_image.shape[0] for boxes_in_image in proposals]
    pred_boxes = self.box_coder.decode(box_regression, proposals)
    pred_scores = F.softmax(class_logits, -1)
    pred_boxes_list = pred_boxes.split(boxes_per_image, 0)
    pred_scores_list = pred_scores.split(boxes_per_image, 0)
    all_boxes, all_scores, all_labels = [], [], []
    for boxes, scores, image_shape in zip(pred_boxes_list, pred_scores_list, image_shapes):
        n = scores.shape[0]
        labels = torch.arange(1, num_classes, device=device).view(1, -1).expand(n, num_classes - 1)
        # background column dropped, every class prediction becomes a separate instance (roi_heads.py:712-721)
        b, s, l = detection_postprocess(boxes[:, 1:].reshape(-1, 4), scores[:, 1:].reshape(-1), labels.reshape(-1), image_shape,
                                        self.score_thresh, False, 1e-2, self.nms_thresh, self.detections_per_img)
        all_boxes.append(b)
        all_scores.append(s)
        all_labels.append(l)
    return all_boxes, all_scores, all_labels


def rpn_filter_proposals(self, proposals, objectness, image_shapes, num_anchors_per_level, _orig=None):
    """RegionProposalNetwork.filter_proposals with the per-image tail fused."""
    if not _fusable(proposals):
        return _orig(self, proposals, objectness, image_shapes, num_anchors_per_level)
    num_images = proposals.shape[0]
    device = proposals.device
    objectness = objectness.detach().reshape(num_images, -1)
    levels = torch.cat([torch.full((n,), idx, dtype=torch.int64, device=device) for idx, n in enumerate(num_anchors_per_level)], 0)
    levels = levels.reshape(1, -1).expand_as(objectness)
    top_n_idx = self._get_top_n_idx(objectness, num_anchors_per_level)
    batch_idx = torch.arange(num_images, device=device)[:, None]
    objectness = objectness[batch_idx, top_n_idx]
    levels = levels[batch_idx, top_n_idx]
    proposals = proposals[batch_idx, top_n_idx]
    objectness_prob = torch.sigmoid(objectness)
    final_boxes, final_scores = [], []
    for boxes, scores, lvl, img_shape in zip(proposals, objectness_prob, levels, image_shapes):
        b, s, _ = detection_postprocess(boxes, scores, lvl, img_shape, self.score_thresh, True, self.min_size, self.nms_thresh,
                                        self.post_nms_top_n())
        final_boxes.append(b)
        final_scores.append(s)
    return final_boxes, final_scores


def _traced() -> bool:
    import torchvision

    return torch.jit.is_scripting() or torch.jit.is_tracing() or torchvision._is_tracing()


def _dense_f32(t) -> bool:
    return isinstance(t, Tensor) and t.is_cuda and t.dtype == torch.float32 and t.dim() >= 2 and t.stride(-1) == 1


def _levels_ok(logits, extra, anchors, num_images: int, extra_width: int) -> bool:
    """Per-level [N, A_l, C] logits, [N, A_l, extra_width] companions and N * L [A_l, 4] anchors, as the kernel takes them;
    a level of 2^31 or more logits is left to the reference (the kernel indexes a segment with 32 bits)."""
    if not isinstance(logits, (list, tuple)) or not logits or len(anchors) != num_images * len(logits):
        return False
    C = logits[0].shape[-1] if isinstance(logits[0], Tensor) else -1
    for l, lg in enumerate(logits):
        if not (_dense_f32(lg) and lg.dim() == 3 and lg.shape[0] == num_images and lg.shape[2] == C and lg.shape[1] * C < 2**31):
            return False
        for t, width in zip(extra[l], extra_width):
            if not (_dense_f32(t) and t.dim() == 3 and tuple(t.shape) == (num_images, lg.shape[1], width)):
                return False
    for i, a in enumerate(anchors):
        if not (_dense_f32(a) and a.dim() == 2 and tuple(a.shape) == (logits[i % len(logits)].shape[1], 4)):
            return False
    return True


def single_stage_postprocess(kind: int, logits, ctrness, regression, anchors, image_shapes, score_thresh: float, topk_candidates: int,
                             nms_thresh: float, detections_per_img: int, weights=(1.0, 1.0, 1.0, 1.0), bbox_xform_clip: float = 0.0):
    """All images of a single-stage detector's postprocess_detections in one call; returns the reference's list of dicts."""
    _lib.load_ops()
    sizes = [int(v) for hw in image_shapes for v in hw]
    boxes, scores, labels, counts = torch.ops.vision_b200.single_stage_postprocess(
        kind, list(logits), list(ctrness), list(regression), list(anchors), sizes, float(score_thresh), int(topk_candidates),
        float(nms_thresh), int(detections_per_img), [float(w) for w in weights], float(bbox_xform_clip))
    counts = counts.tolist()
    return [{"boxes": b, "scores": s, "labels": l}
            for b, s, l in zip(boxes.split(counts), scores.split(counts), labels.split(counts))]


def retinanet_postprocess_detections(self, head_outputs, anchors, image_shapes, _orig=None):
    """RetinaNet.postprocess_detections as one fused call (same outputs, same order)."""
    from torchvision.models.detection import _utils as det_utils

    logits, regression = head_outputs["cls_logits"], head_outputs["bbox_regression"]
    flat_anchors = [a for per_image in anchors for a in per_image]
    if (_traced() or type(self.box_coder) is not det_utils.BoxCoder or not 0 <= self.topk_candidates <= SINGLE_STAGE_MAX_TOPK
            or len(regression) != len(logits) or len(anchors) != len(image_shapes)
            or not _levels_ok(logits, [(r,) for r in regression], flat_anchors, len(image_shapes), (4,))):
        return _orig(self, head_outputs, anchors, image_shapes)
    coder = self.box_coder
    return single_stage_postprocess(_SS_RETINANET, logits, [], regression, flat_anchors, image_shapes, self.score_thresh,
                                    self.topk_candidates, self.nms_thresh, self.detections_per_img, coder.weights, coder.bbox_xform_clip)


def fcos_postprocess_detections(self, head_outputs, anchors, image_shapes, _orig=None):
    """FCOS.postprocess_detections as one fused call (same outputs, same order)."""
    from torchvision.models.detection import _utils as det_utils

    logits, regression, ctrness = head_outputs["cls_logits"], head_outputs["bbox_regression"], head_outputs["bbox_ctrness"]
    flat_anchors = [a for per_image in anchors for a in per_image]
    if (_traced() or type(self.box_coder) is not det_utils.BoxLinearCoder or self.box_coder.normalize_by_size is not True
            or not 0 <= self.topk_candidates <= SINGLE_STAGE_MAX_TOPK or len(regression) != len(logits) or len(ctrness) != len(logits)
            or len(anchors) != len(image_shapes)
            or not _levels_ok(logits, list(zip(regression, ctrness)), flat_anchors, len(image_shapes), (4, 1))):
        return _orig(self, head_outputs, anchors, image_shapes)
    return single_stage_postprocess(_SS_FCOS, logits, ctrness, regression, flat_anchors, image_shapes, self.score_thresh,
                                    self.topk_candidates, self.nms_thresh, self.detections_per_img)


def ssd_postprocess_detections(self, head_outputs, image_anchors, image_shapes, _orig=None):
    """SSD.postprocess_detections (also SSDLite) as softmax + one fused call (same outputs, same order)."""
    from torchvision.models.detection import _utils as det_utils

    logits, regression = head_outputs["cls_logits"], head_outputs["bbox_regression"]
    if (_traced() or type(self.box_coder) is not det_utils.BoxCoder or not 0 <= self.topk_candidates <= SINGLE_STAGE_MAX_TOPK
            or not isinstance(image_anchors, (list, tuple)) or len(image_anchors) != len(image_shapes)
            or not _levels_ok([logits], [(regression,)], list(image_anchors), len(image_shapes), (4,))):
        return _orig(self, head_outputs, image_anchors, image_shapes)
    pred_scores = F.softmax(logits, dim=-1)          # ssd.py:418
    coder = self.box_coder
    return single_stage_postprocess(_SS_SSD, [pred_scores], [], [regression], image_anchors, image_shapes, self.score_thresh,
                                    self.topk_candidates, self.nms_thresh, self.detections_per_img, coder.weights, coder.bbox_xform_clip)


# largest heatmap side the keypoint kernel stages in shared memory (VB200_KP_MAX_SIDE in include/vision_b200.h)
KEYPOINTS_MAX_SIDE = 128


def keypoints_supported(maps, rois) -> bool:
    """Inputs the keypoint kernel takes: CUDA fp32 / fp16 / bf16 maps [K, N, H, W] with H, W <= KEYPOINTS_MAX_SIDE, fp32 rois
    [K, 4] on the same device, outside scripting and tracing (the reference keeps its ONNX loop there)."""
    return (isinstance(maps, Tensor) and isinstance(rois, Tensor) and maps.is_cuda and rois.is_cuda and maps.device == rois.device
            and maps.dtype in (torch.float32, torch.float16, torch.bfloat16) and maps.dim() == 4 and rois.dtype == torch.float32
            and rois.dim() == 2 and rois.shape[1] == 4 and maps.shape[0] == rois.shape[0] and maps.shape[1] >= 1
            and 1 <= maps.shape[2] <= KEYPOINTS_MAX_SIDE and 1 <= maps.shape[3] <= KEYPOINTS_MAX_SIDE and not _traced())


def _boxes_sized(rois: Tensor) -> bool:
    """The one host read-back of a call: every box's resized map has a finite size below 2^31 pixels.  The others go to the
    reference body, which raises (a NaN or infinite size) or behaves as it does today.  fp32 rounds the product up, never
    down, across 2^31, so no box past the limit passes."""
    wh = (rois[:, 2:] - rois[:, :2]).clamp(min=1).ceil()
    return bool((wh[:, 0] * wh[:, 1] < 2.0**31).all())


def heatmaps_to_keypoints_op(maps: Tensor, rois: Tensor):
    _lib.load_ops()
    return torch.ops.vision_b200.heatmaps_to_keypoints(maps, rois)


def heatmaps_to_keypoints(maps, rois, _orig=None):
    """roi_heads.heatmaps_to_keypoints as one fused call (same outputs, shapes and strides)."""
    if not (keypoints_supported(maps, rois) and _boxes_sized(rois)):
        return _orig(maps, rois)
    return heatmaps_to_keypoints_op(maps, rois)


def keypointrcnn_inference(x, boxes, _orig=None):
    """roi_heads.keypointrcnn_inference with every image's heatmaps_to_keypoints in ONE call: the boxes concatenated, one op,
    per-image views of its outputs."""
    if not (isinstance(boxes, (list, tuple)) and boxes
            and all(isinstance(b, Tensor) and b.is_cuda and b.dtype == torch.float32 for b in boxes)):
        return _orig(x, boxes)
    rois = torch.cat(list(boxes)) if len(boxes) > 1 else boxes[0]
    if not (keypoints_supported(x, rois) and _boxes_sized(rois)):
        return _orig(x, boxes)
    xy, scores = heatmaps_to_keypoints_op(x, rois)
    counts = [b.size(0) for b in boxes]
    return list(xy.split(counts)), list(scores.split(counts))


_RCNN_DTYPES = (torch.float32, torch.float16, torch.bfloat16)
_RCNN_MAX_CHANNELS = 8
_RCNN_MAX_PAD_H = 65535 * 8          # rows of the batch kernel's grid: 65535 tiles of 8


def rcnn_output_size(h: int, w: int, min_size, max_size, fixed_size):
    """The size _resize_image_and_masks (transform.py:25-72) resizes an h x w image to in eval mode: fixed_size reversed, or
    F.interpolate's recompute_scale_factor rule, int(side * scale) with the scale in Python double."""
    if fixed_size is not None:
        return int(fixed_size[1]), int(fixed_size[0])
    scale = min(min_size / min(h, w), max_size / max(h, w))
    return int(h * scale), int(w * scale)


def _rcnn_batch_plan(self, images):
    """The per-image output sizes and the padded size when the batch kernel reproduces the reference's forward for these
    images, else None.  Inference only, outside deterministic mode (F.interpolate decomposes there), scripting and
    tracing; CUDA images [C, H, W] of one dtype (fp32, or fp16 / bf16 with autocast off), device and channel count, one
    mean and std per channel (the reference broadcasts others), output sides >= 1 and planes below 2^31 elements."""
    if (self.training or torch.are_deterministic_algorithms_enabled() or _traced() or not images
            or not all(isinstance(img, Tensor) for img in images)):
        return None
    i0 = images[0]
    if not (i0.is_cuda and i0.dtype in _RCNN_DTYPES and i0.dim() == 3):
        return None
    if i0.dtype != torch.float32 and torch.is_autocast_enabled("cuda"):
        return None
    C = i0.shape[0]
    if not (1 <= C <= _RCNN_MAX_CHANNELS and len(self.image_mean) == C and len(self.image_std) == C):
        return None
    sizes = []
    for img in images:
        if not (img.device == i0.device and img.dtype == i0.dtype and img.dim() == 3 and img.shape[0] == C):
            return None
        h, w = img.shape[-2:]
        if h < 1 or w < 1 or h * w >= 2**31:
            return None
        oh, ow = rcnn_output_size(h, w, self.min_size[-1], self.max_size, self.fixed_size)
        if oh < 1 or ow < 1 or oh * ow >= 2**31:
            return None
        sizes.append((oh, ow))
    stride = float(self.size_divisible)          # batch_images (transform.py:243-247)
    pad_h = int(math.ceil(float(max(s[0] for s in sizes)) / stride) * stride)
    pad_w = int(math.ceil(float(max(s[1] for s in sizes)) / stride) * stride)
    if pad_h > _RCNN_MAX_PAD_H or pad_h * pad_w >= 2**31:
        return None
    return sizes, pad_h, pad_w


def rcnn_batch_images_op(images, out_sizes, pad_h: int, pad_w: int, mean, std) -> Tensor:
    _lib.load_ops()
    return torch.ops.vision_b200.rcnn_batch_images(list(images), [s[0] for s in out_sizes], [s[1] for s in out_sizes], pad_h, pad_w,
                                                   list(mean), list(std))


def rcnn_transform_forward(self, images, targets=None, _orig=None):
    """GeneralizedRCNNTransform.forward in eval mode as one fused call: the same ImageList (padded batch and image_sizes as
    tuples of Python ints) and targets None.  Training, targets and inputs the kernel does not cover run the reference."""
    from torchvision.models.detection.image_list import ImageList

    imgs = [img for img in images] if isinstance(images, (list, tuple, Tensor)) else None
    plan = _rcnn_batch_plan(self, imgs) if targets is None and imgs is not None else None
    if plan is None:
        return _orig(self, images, targets)
    sizes, pad_h, pad_w = plan
    # mean and std exactly as normalize's torch.as_tensor(list, dtype=dtype) rounds them (transform.py:167-168)
    mean = torch.as_tensor(self.image_mean, dtype=imgs[0].dtype).tolist()
    std = torch.as_tensor(self.image_std, dtype=imgs[0].dtype).tolist()
    batched = rcnn_batch_images_op(imgs, sizes, pad_h, pad_w, mean, std)
    return ImageList(batched, [(int(h), int(w)) for h, w in sizes]), None


def _rcnn_ratios(new_size, original_size):
    """resize_boxes / resize_keypoints' ratios (transform.py:289-294, 307-312): fp32 new / original, (height, width)."""
    q = np.float32(new_size) / np.float32(original_size) if all(o != 0 for o in original_size) else None
    return None if q is None else (float(q[0]), float(q[1]))


def rcnn_rescale_op(inputs, ratio_w, ratio_h):
    _lib.load_ops()
    return torch.ops.vision_b200.rcnn_rescale(list(inputs), list(ratio_w), list(ratio_h))


def rcnn_transform_postprocess(self, result, image_shapes, original_image_sizes, _orig=None):
    """GeneralizedRCNNTransform.postprocess in eval mode with every image's boxes and keypoints rescaled by one fused call;
    masks are pasted by the reference's paste_masks_in_image with the rescaled boxes.  Same dicts, updated in place."""
    from torchvision.models.detection import transform as tv_transform

    if self.training or _traced() or not isinstance(result, (list, tuple)):
        return _orig(self, result, image_shapes, original_image_sizes)
    triples = list(zip(result, image_shapes, original_image_sizes))
    inputs, rw, rh, slots = [], [], [], []
    for i, (pred, im_s, o_im_s) in enumerate(triples):
        boxes = pred.get("boxes") if isinstance(pred, dict) else None
        ratios = _rcnn_ratios(o_im_s, im_s) if len(im_s) == 2 and len(o_im_s) == 2 else None
        if not (isinstance(boxes, Tensor) and boxes.is_cuda and boxes.dtype == torch.float32 and boxes.dim() == 2
                and boxes.shape[1] == 4 and ratios is not None):
            return _orig(self, result, image_shapes, original_image_sizes)
        named = [("boxes", boxes)]
        if "keypoints" in pred:
            kp = pred["keypoints"]
            if not (isinstance(kp, Tensor) and kp.is_cuda and kp.dtype == torch.float32 and kp.dim() == 3 and kp.shape[2] == 3):
                return _orig(self, result, image_shapes, original_image_sizes)
            named.append(("keypoints", kp))
        for key, t in named:
            if t.device != boxes.device or (inputs and t.device != inputs[0].device):
                return _orig(self, result, image_shapes, original_image_sizes)
            inputs.append(t)
            rh.append(ratios[0])
            rw.append(ratios[1])
            slots.append((i, key))
    if not inputs:
        return result
    outs = rcnn_rescale_op(inputs, rw, rh)
    for (i, key), out in zip(slots, outs):
        result[i][key] = out
    for i, (pred, im_s, o_im_s) in enumerate(triples):
        if "masks" in pred:
            result[i]["masks"] = tv_transform.paste_masks_in_image(pred["masks"], result[i]["boxes"], o_im_s)
    return result


MATCH_RAW, MATCH_RPN, MATCH_ROI_HEADS = 0, 1, 2          # VB200_MATCH_* in include/vision_b200.h
_MATCH_DTYPES = (torch.float16, torch.bfloat16, torch.float32, torch.float64)


def match_supported(matcher, gt_boxes, predictions, gt_labels=None) -> bool:
    """Inputs the matching kernel reproduces the reference on: a plain ``det_utils.Matcher`` (not SSD's SSDMatcher or a
    subclass) with its -1 / -2 codes, outside scripting and tracing; one [M, 4] gt (or an empty one: a background image)
    and one [N, 4] prediction tensor per image, N below 2^31, all CUDA on one device; the gt boxes that have elements of one
    dtype and the predictions of one dtype, both fp64 or both among fp16 / bf16 / fp32; for RoIHeads, int64 [M] labels."""
    from torchvision.models.detection import _utils as det_utils

    if type(matcher) is not det_utils.Matcher or matcher.BELOW_LOW_THRESHOLD != -1 or matcher.BETWEEN_THRESHOLDS != -2:
        return False
    return _box_lists_supported(gt_boxes, predictions, gt_labels)


def _box_lists_supported(gt_boxes, predictions, gt_labels=None) -> bool:
    """The per-image box lists both matching kernels take (see match_supported), outside scripting and tracing."""
    if (_traced() or not isinstance(gt_boxes, (list, tuple)) or not isinstance(predictions, (list, tuple)) or not predictions
            or len(gt_boxes) != len(predictions) or (gt_labels is not None and len(gt_labels) != len(predictions))):
        return False
    p0 = predictions[0]
    if not (isinstance(p0, Tensor) and p0.is_cuda and p0.dtype in _MATCH_DTYPES):
        return False
    gdt = None
    for i, (g, p) in enumerate(zip(gt_boxes, predictions)):
        if not (isinstance(g, Tensor) and isinstance(p, Tensor) and p.is_cuda and p.device == p0.device and p.dtype == p0.dtype
                and p.dim() == 2 and p.shape[1] == 4 and p.shape[0] < 2**31):
            return False
        if g.numel() == 0:
            continue
        if not (g.is_cuda and g.device == p0.device and g.dim() == 2 and g.shape[1] == 4 and g.dtype in _MATCH_DTYPES
                and g.dtype == (gdt or g.dtype) and (g.dtype == torch.float64) == (p.dtype == torch.float64)):
            return False
        gdt = g.dtype
        if gt_labels is not None:
            lb = gt_labels[i]
            if not (isinstance(lb, Tensor) and lb.is_cuda and lb.device == p0.device and lb.dtype == torch.int64
                    and tuple(lb.shape) == (g.shape[0],)):
                return False
    return True


def match_boxes_op(gt_boxes, predictions, gt_labels, matcher, mode: int):
    """Every image's box_iou + Matcher + the caller's epilogue as one op.  An image with gt boxes and no predictions raises
    the Matcher's error from the shapes, before anything is launched."""
    for g, p in zip(gt_boxes, predictions):
        if g.numel() != 0 and p.shape[0] == 0:
            raise ValueError("No proposal boxes available for one of the images during training")
    _lib.load_ops()
    return torch.ops.vision_b200.match_boxes(list(gt_boxes), list(predictions), list(gt_labels or []), float(matcher.high_threshold),
                                             float(matcher.low_threshold), bool(matcher.allow_low_quality_matches), mode)


def rpn_assign_targets_to_anchors(self, anchors, targets, _orig=None):
    """RegionProposalNetwork.assign_targets_to_anchors as one fused call: the same fp32 labels and matched gt boxes."""
    from torchvision.ops import boxes as box_ops

    gt_boxes = [t["boxes"] for t in targets] if isinstance(targets, (list, tuple)) else None
    if self.box_similarity is not box_ops.box_iou or gt_boxes is None or not match_supported(self.proposal_matcher, gt_boxes, anchors):
        return _orig(self, anchors, targets)
    return match_boxes_op(gt_boxes, anchors, None, self.proposal_matcher, MATCH_RPN)


def roi_heads_assign_targets_to_proposals(self, proposals, gt_boxes, gt_labels, _orig=None):
    """RoIHeads.assign_targets_to_proposals as one fused call: the same clamped matches and int64 labels."""
    if not match_supported(self.proposal_matcher, gt_boxes, proposals, gt_labels):
        return _orig(self, proposals, gt_boxes, gt_labels)
    return match_boxes_op(gt_boxes, proposals, gt_labels, self.proposal_matcher, MATCH_ROI_HEADS)


def retinanet_compute_loss(self, targets, head_outputs, anchors, _orig=None):
    """RetinaNet.compute_loss with its matching loop as one fused call; self.head.compute_loss is the reference's."""
    gt_boxes = [t["boxes"] for t in targets] if isinstance(targets, (list, tuple)) else None
    if gt_boxes is None or not match_supported(self.proposal_matcher, gt_boxes, anchors):
        return _orig(self, targets, head_outputs, anchors)
    matched_idxs, _ = match_boxes_op(gt_boxes, anchors, None, self.proposal_matcher, MATCH_RAW)
    return self.head.compute_loss(targets, head_outputs, anchors, matched_idxs)


def _same_gpu(t, device, dtype=None, dim=None) -> bool:
    return (isinstance(t, Tensor) and t.is_cuda and t.device == device and (dtype is None or t.dtype == dtype)
            and (dim is None or t.dim() == dim))


def _loss_inputs_ok(targets, pred, matched_idxs, width) -> bool:
    """What both fused head losses take: outside scripting and tracing, one target dict and one int64 [A] matched_idxs per
    image of a fp32 CUDA [B, A, width] prediction tensor whose rows are dense, A * width below 2^31."""
    if (_traced() or not isinstance(targets, (list, tuple)) or not targets or not isinstance(matched_idxs, (list, tuple))
            or not isinstance(pred, Tensor) or not pred.is_cuda or pred.dtype != torch.float32 or pred.dim() != 3):
        return False
    B, A, C = pred.shape
    if not (len(targets) == len(matched_idxs) == B and C == width >= 1 and A * C < 2**31 and pred.stride(2) == 1
            and (A <= 1 or pred.stride(1) == C)):
        return False
    return all(isinstance(t, dict) and _same_gpu(m, pred.device, torch.int64, 1) and m.shape[0] == A
               for t, m in zip(targets, matched_idxs))


def retinanet_cls_loss_supported(head, targets, cls_logits, matched_idxs) -> bool:
    """Inputs the focal-loss kernels reproduce RetinaNetClassificationHead.compute_loss on: those of _loss_inputs_ok with
    the logits' C, an int64 [M] labels tensor per image on the logits' GPU, and the Matcher's -2 for ignored anchors."""
    if getattr(head, "BETWEEN_THRESHOLDS", None) != -2 or not isinstance(cls_logits, Tensor) or cls_logits.dim() != 3:
        return False
    if not _loss_inputs_ok(targets, cls_logits, matched_idxs, cls_logits.shape[2]):
        return False
    return all(_same_gpu(t.get("labels"), cls_logits.device, torch.int64, 1) for t in targets)


def retinanet_cls_loss_op(cls_logits, matched_idxs, labels):
    _lib.load_ops()
    loss, _ = torch.ops.vision_b200.retinanet_cls_loss(cls_logits, list(matched_idxs), list(labels))
    return loss


def retinanet_cls_compute_loss(self, targets, head_outputs, matched_idxs, _orig=None):
    """RetinaNetClassificationHead.compute_loss as one fused call for all images: the same loss, and a dense gradient of
    cls_logits written in one pass."""
    cls_logits = head_outputs["cls_logits"] if isinstance(head_outputs, dict) else None
    if not retinanet_cls_loss_supported(self, targets, cls_logits, matched_idxs):
        return _orig(self, targets, head_outputs, matched_idxs)
    return retinanet_cls_loss_op(cls_logits, matched_idxs, [t["labels"] for t in targets])


def _coder_weights(box_coder):
    """The coder's weights as encode_single's torch.as_tensor(weights, dtype=float32) rounds them, or None."""
    w = box_coder.weights
    if not isinstance(w, (list, tuple)) or len(w) != 4 or not all(isinstance(v, (int, float)) for v in w):
        return None
    return [float(v) for v in np.asarray(w, dtype=np.float32)]


def retinanet_box_loss_supported(head, targets, bbox_regression, anchors, matched_idxs) -> bool:
    """Inputs the box-loss kernels reproduce RetinaNetRegressionHead.compute_loss on: the "l1" loss with a plain
    ``det_utils.BoxCoder`` of four numeric weights, the inputs of _loss_inputs_ok with width 4, and fp32 [A, 4] anchors and
    [M, 4] gt boxes per image on the regression's GPU."""
    from torchvision.models.detection import _utils as det_utils

    if getattr(head, "_loss_type", None) != "l1" or type(getattr(head, "box_coder", None)) is not det_utils.BoxCoder:
        return False
    if _coder_weights(head.box_coder) is None or not _loss_inputs_ok(targets, bbox_regression, matched_idxs, 4):
        return False
    if not isinstance(anchors, (list, tuple)) or len(anchors) != len(targets):
        return False
    A, device = bbox_regression.shape[1], bbox_regression.device
    for t, a in zip(targets, anchors):
        g = t.get("boxes")
        if not (_same_gpu(g, device, torch.float32, 2) and g.shape[1] == 4 and _same_gpu(a, device, torch.float32, 2)
                and tuple(a.shape) == (A, 4)):
            return False
    return True


def retinanet_box_loss_op(bbox_regression, anchors, gt_boxes, matched_idxs, weights):
    _lib.load_ops()
    loss, _ = torch.ops.vision_b200.retinanet_box_loss(bbox_regression, list(anchors), list(gt_boxes), list(matched_idxs), list(weights))
    return loss


def retinanet_box_compute_loss(self, targets, head_outputs, anchors, matched_idxs, _orig=None):
    """RetinaNetRegressionHead.compute_loss ("l1") as one fused call for all images: the same loss, and a dense gradient of
    bbox_regression written in one pass."""
    regression = head_outputs["bbox_regression"] if isinstance(head_outputs, dict) else None
    if not retinanet_box_loss_supported(self, targets, regression, anchors, matched_idxs):
        return _orig(self, targets, head_outputs, anchors, matched_idxs)
    return retinanet_box_loss_op(regression, anchors, [t["boxes"] for t in targets], matched_idxs, _coder_weights(self.box_coder))


def fcos_match_supported(gt_boxes, anchors, num_anchors_per_level, radius) -> bool:
    """Inputs the FCOS kernel reproduces the reference on: the box lists of match_supported (one [M, 4] gt, or one without
    elements, and one [N, 4] anchor tensor per image, N below 2^31, all CUDA on one device, the gt of one dtype and the
    anchors of one, both fp64 or both among fp16 / bf16 / fp32), outside scripting and tracing; a non-empty
    num_anchors_per_level whose first and last entries are ints; a real center_sampling_radius."""
    return (isinstance(num_anchors_per_level, (list, tuple)) and len(num_anchors_per_level) > 0
            and all(isinstance(k, int) and abs(k) < 2**62 for k in (num_anchors_per_level[0], num_anchors_per_level[-1]))
            and isinstance(radius, (int, float)) and _box_lists_supported(gt_boxes, anchors))


def fcos_match_op(gt_boxes, anchors, radius, num_anchors_per_level):
    """Every image's matched_idx of FCOS.compute_loss (fcos.py:447-485) as one op: int64 [N] per image, -1 unmatched."""
    _lib.load_ops()
    return torch.ops.vision_b200.fcos_match(list(gt_boxes), list(anchors), float(radius), int(num_anchors_per_level[0]),
                                            int(num_anchors_per_level[-1]))


def fcos_compute_loss(self, targets, head_outputs, anchors, num_anchors_per_level, _orig=None):
    """FCOS.compute_loss with its matching loop as one fused call; self.head.compute_loss is the reference's."""
    gt_boxes = [t["boxes"] for t in targets] if isinstance(targets, (list, tuple)) else None
    if gt_boxes is None or not fcos_match_supported(gt_boxes, anchors, num_anchors_per_level, self.center_sampling_radius):
        return _orig(self, targets, head_outputs, anchors, num_anchors_per_level)
    matched_idxs = fcos_match_op(gt_boxes, anchors, self.center_sampling_radius, num_anchors_per_level)
    return self.head.compute_loss(targets, head_outputs, anchors, matched_idxs)
