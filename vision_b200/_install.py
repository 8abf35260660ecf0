"""install()/uninstall(): put the kernels behind torchvision's own API surface.

1. dispatcher ops (nms, roi_align, roi_pool, ps_roi_align, deform_conv2d): re-registered for the
   CUDA key of the existing ``torchvision::`` schemas by the C++ shim (a run-time twin of the
   reference's TORCH_LIBRARY_IMPL blocks, e.g. csrc/ops/cuda/roi_align_kernel.cu:470-477).  Meta,
   Autograd, Autocast, CPU and quantized registrations are untouched.
2. ``batched_nms`` is Python in the reference (torchvision/ops/boxes.py:57-126): the module
   attribute is rebound (detection models call ``box_ops.batched_nms`` at call time).
3. ``MultiScaleRoIAlign`` (torchvision/ops/poolers.py:147-228): the module-level ``_multiscale_roi_align`` is rebound
   to the fused kernel (device-side LevelMapper + one gather launch over all FPN levels) when the shape is covered.
   ``torchvision.ops.roi_align``'s deterministic-mode route (a compiled pure-PyTorch roi_align) is rebound to the
   dispatcher op, whose backward is bit-reproducible in that mode.
4. detection post-processing: ``RoIHeads.postprocess_detections`` and ``RegionProposalNetwork.filter_proposals`` keep their
   tensor prologue and run the per-image tail (clip, filters, batched_nms, top-k, gathers) as one fused call;
   ``RetinaNet``, ``FCOS`` and ``SSD`` (and so SSDLite) ``postprocess_detections`` run as one fused call for all images;
   the module globals ``roi_heads.keypointrcnn_inference`` and ``roi_heads.heatmaps_to_keypoints`` (Keypoint R-CNN) are
   rebound to one keypoint-extraction call for all images.
   ``GeneralizedRCNNTransform.forward`` and ``.postprocess``, which every detection model enters and leaves through, are
   rebound on the class: normalize, resize and padding of all images in one call, the rescaling of every image's boxes and
   keypoints in another.
   Training targets: ``RegionProposalNetwork.assign_targets_to_anchors``, ``RoIHeads.assign_targets_to_proposals`` and
   ``RetinaNet.compute_loss`` are rebound on their classes; the per-image box_iou + Matcher loop becomes one call.
   ``FCOS.compute_loss`` likewise: its per-image centre-sampling loop becomes one call.
   Head losses: ``RetinaNetClassificationHead.compute_loss`` and ``RetinaNetRegressionHead.compute_loss`` are rebound on
   their classes; each per-image loss loop becomes one call with a fused backward.  ``FCOSHead.compute_loss`` likewise:
   its three losses become two calls, each with a fused backward.  The module global ``roi_heads.maskrcnn_loss`` (Mask
   R-CNN) is rebound to one mask-loss call for all images with a fused backward.
5. ``resize`` has no torchvision kernel (transforms/v2/functional/_geometry.py:283-362 calls
   F.interpolate): the entries of ``_KERNEL_REGISTRY[resize]`` for Tensor / Image / Video are swapped.
CPU tensors and unsupported dtypes/modes keep flowing to the reference implementation.
"""
from __future__ import annotations

import functools
import warnings

import torch

from . import _lib, transforms as _tf

_state: dict = {}


def installed() -> bool:
    return bool(_state)


def install() -> None:
    if _state:
        return
    import torchvision  # the schemas must exist before the CUDA key is overridden
    from torchvision.ops import boxes as tv_boxes
    from torchvision.transforms.v2.functional import _geometry as tv_geo, _utils as tv_utils
    from torchvision import tv_tensors

    _lib.load_ops()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")   # "Overriding a previously registered kernel" (expected)
        torch.ops.vision_b200._install(True)

    # ---- batched_nms ----
    orig_batched_nms = tv_boxes.batched_nms

    @functools.wraps(orig_batched_nms)
    def batched_nms(boxes, scores, idxs, iou_threshold):
        if (isinstance(boxes, torch.Tensor) and boxes.is_cuda and boxes.dtype in (torch.float32, torch.float64, torch.float16)
                and not torch.jit.is_scripting() and not torch.jit.is_tracing()):
            return torch.ops.vision_b200.batched_nms(boxes, scores, idxs, float(iou_threshold))
        return orig_batched_nms(boxes, scores, idxs, iou_threshold)

    tv_boxes.batched_nms = batched_nms
    torchvision.ops.batched_nms = batched_nms

    # ---- MultiScaleRoIAlign: the per-level loop of poolers.py:147-228 becomes one fused call when the kernel covers it ----
    from torchvision.ops import poolers as tv_poolers
    from . import ops as _ops_mod

    orig_msra = tv_poolers._multiscale_roi_align

    def _multiscale_roi_align(x_filtered, boxes, output_size, sampling_ratio, scales, mapper):
        if (scales is not None and mapper is not None and not torch.jit.is_scripting() and not torch.jit.is_tracing()
                and not torchvision._is_tracing() and _ops_mod.multiscale_roi_align_supported(x_filtered, boxes, output_size, sampling_ratio)):
            return _ops_mod.multiscale_roi_align(x_filtered, boxes, output_size, sampling_ratio, scales, mapper)
        return orig_msra(x_filtered, boxes, output_size, sampling_ratio, scales, mapper)

    tv_poolers._multiscale_roi_align = _multiscale_roi_align

    # ---- roi_align under torch.use_deterministic_algorithms (roi_align.py:250-256): torchvision sends CUDA inputs to a
    # torch.compile'd pure-PyTorch roi_align, since its own backward is atomic.  Ours is bit-reproducible in that mode, so
    # the route is rebound to the dispatcher op.  torchvision's lazy compile rebinds the name on its first call, so the
    # fall-back puts ours back afterwards.
    import sys

    tv_roi_align_mod = sys.modules["torchvision.ops.roi_align"]
    orig_det_roi_align = tv_roi_align_mod._roi_align

    def _roi_align(input, rois, spatial_scale, pooled_height, pooled_width, sampling_ratio, aligned):
        if input.is_cuda and input.dtype in (torch.float32, torch.float64, torch.float16):
            return torch.ops.torchvision.roi_align(input, rois, spatial_scale, pooled_height, pooled_width, sampling_ratio, aligned)
        try:
            return orig_det_roi_align(input, rois, spatial_scale, pooled_height, pooled_width, sampling_ratio, aligned)
        finally:
            tv_roi_align_mod._roi_align = _roi_align

    tv_roi_align_mod._roi_align = _roi_align

    # ---- detection post-processing around batched_nms (roi_heads.py:680-737, rpn.py:242-298) ----
    from torchvision.models.detection import roi_heads as tv_roi_heads, rpn as tv_rpn
    from . import detection as _det

    orig_pp = tv_roi_heads.RoIHeads.postprocess_detections
    orig_fp = tv_rpn.RegionProposalNetwork.filter_proposals

    def postprocess_detections(self, class_logits, box_regression, proposals, image_shapes):
        if _det._fusable(class_logits) and not torchvision._is_tracing():
            return _det.roi_heads_postprocess_detections(self, class_logits, box_regression, proposals, image_shapes, _orig=orig_pp)
        return orig_pp(self, class_logits, box_regression, proposals, image_shapes)

    def filter_proposals(self, proposals, objectness, image_shapes, num_anchors_per_level):
        if _det._fusable(proposals) and not torchvision._is_tracing():
            return _det.rpn_filter_proposals(self, proposals, objectness, image_shapes, num_anchors_per_level, _orig=orig_fp)
        return orig_fp(self, proposals, objectness, image_shapes, num_anchors_per_level)

    tv_roi_heads.RoIHeads.postprocess_detections = postprocess_detections
    tv_rpn.RegionProposalNetwork.filter_proposals = filter_proposals

    # ---- Keypoint R-CNN inference (roi_heads.py:237-354): RoIHeads.forward looks up keypointrcnn_inference at call time ----
    orig_kri = tv_roi_heads.keypointrcnn_inference
    orig_h2k = tv_roi_heads.heatmaps_to_keypoints

    @functools.wraps(orig_kri)
    def keypointrcnn_inference(x, boxes):
        return _det.keypointrcnn_inference(x, boxes, _orig=orig_kri)

    @functools.wraps(orig_h2k)
    def heatmaps_to_keypoints(maps, rois):
        return _det.heatmaps_to_keypoints(maps, rois, _orig=orig_h2k)

    tv_roi_heads.keypointrcnn_inference = keypointrcnn_inference
    tv_roi_heads.heatmaps_to_keypoints = heatmaps_to_keypoints

    # ---- training-target assignment (rpn.py:193-229, roi_heads.py:580-613, retinanet.py:494-507, fcos.py:440-487): bound on
    # the classes ----
    from torchvision.models.detection import fcos as tv_fcos, retinanet as tv_retinanet

    matching = {}
    for cls, name, body in ((tv_rpn.RegionProposalNetwork, "assign_targets_to_anchors", _det.rpn_assign_targets_to_anchors),
                            (tv_roi_heads.RoIHeads, "assign_targets_to_proposals", _det.roi_heads_assign_targets_to_proposals),
                            (tv_retinanet.RetinaNet, "compute_loss", _det.retinanet_compute_loss),
                            (tv_fcos.FCOS, "compute_loss", _det.fcos_compute_loss)):
        orig = getattr(cls, name)

        def fused(self, *args, _body=body, _orig=orig, **kwargs):
            return _body(self, *args, _orig=_orig, **kwargs)

        functools.update_wrapper(fused, orig)
        matching[(cls, name)] = orig
        setattr(cls, name, fused)

    # ---- RetinaNet head losses (retinanet.py:158-189, 272-302): bound on the head classes; RetinaNetHead.compute_loss stays
    # torchvision's and calls them ----
    losses = {}
    for cls, body in ((tv_retinanet.RetinaNetClassificationHead, _det.retinanet_cls_compute_loss),
                      (tv_retinanet.RetinaNetRegressionHead, _det.retinanet_box_compute_loss)):
        orig = cls.compute_loss

        def fused(self, *args, _body=body, _orig=orig, **kwargs):
            return _body(self, *args, _orig=_orig, **kwargs)

        functools.update_wrapper(fused, orig)
        losses[(cls, "compute_loss")] = orig
        cls.compute_loss = fused

    # ---- FCOS head loss (fcos.py:52-125): bound on FCOSHead; FCOS.compute_loss (its matching fused above) calls it ----
    orig_fcos_head_loss = tv_fcos.FCOSHead.compute_loss

    @functools.wraps(orig_fcos_head_loss)
    def fcos_head_loss(self, targets, head_outputs, anchors, matched_idxs):
        return _det.fcos_head_compute_loss(self, targets, head_outputs, anchors, matched_idxs, _orig=orig_fcos_head_loss)

    tv_fcos.FCOSHead.compute_loss = fcos_head_loss
    fcos_losses = {(tv_fcos.FCOSHead, "compute_loss"): orig_fcos_head_loss}

    # ---- Mask R-CNN mask loss (roi_heads.py:100-129): RoIHeads.forward looks up maskrcnn_loss at call time ----
    orig_mask_loss = tv_roi_heads.maskrcnn_loss

    @functools.wraps(orig_mask_loss)
    def maskrcnn_loss(mask_logits, proposals, gt_masks, gt_labels, mask_matched_idxs):
        return _det.maskrcnn_loss(mask_logits, proposals, gt_masks, gt_labels, mask_matched_idxs, _orig=orig_mask_loss)

    tv_roi_heads.maskrcnn_loss = maskrcnn_loss

    # ---- detection model inputs and outputs (transform.py:119-158, 257-277): bound on the class, so every model's
    # self.transform (Faster / Mask / Keypoint R-CNN, RetinaNet, FCOS, SSD, SSDLite) picks them up ----
    from torchvision.models.detection import transform as tv_transform

    rcnn_transform = tv_transform.GeneralizedRCNNTransform
    orig_tf_forward, orig_tf_post = rcnn_transform.forward, rcnn_transform.postprocess

    @functools.wraps(orig_tf_forward)
    def transform_forward(self, images, targets=None):
        return _det.rcnn_transform_forward(self, images, targets, _orig=orig_tf_forward)

    @functools.wraps(orig_tf_post)
    def transform_postprocess(self, result, image_shapes, original_image_sizes):
        return _det.rcnn_transform_postprocess(self, result, image_shapes, original_image_sizes, _orig=orig_tf_post)

    rcnn_transform.forward = transform_forward
    rcnn_transform.postprocess = transform_postprocess

    # ---- single-stage detectors (retinanet.py:509-571, fcos.py:489-556, ssd.py:414-463) ----
    from torchvision.models.detection import fcos as tv_fcos, retinanet as tv_retinanet, ssd as tv_ssd

    single_stage = {}
    for cls, body in ((tv_retinanet.RetinaNet, _det.retinanet_postprocess_detections), (tv_fcos.FCOS, _det.fcos_postprocess_detections),
                      (tv_ssd.SSD, _det.ssd_postprocess_detections)):
        orig = cls.postprocess_detections

        def fused(self, head_outputs, anchors, image_shapes, _body=body, _orig=orig):
            return _body(self, head_outputs, anchors, image_shapes, _orig=_orig)

        functools.update_wrapper(fused, orig)
        single_stage[cls] = orig
        cls.postprocess_detections = fused

    # ---- ImageClassification preset (transforms/_presets.py:57-64): resize + center_crop + to float + normalize fused ----
    from torchvision.transforms import _presets as tv_presets

    orig_preset_forward = tv_presets.ImageClassification.forward

    def preset_forward(self, img):
        if _tf.classification_preprocess_supported(img, self.crop_size, self.resize_size, self.interpolation, self.antialias):
            return _tf.classification_preprocess(img, self.crop_size, self.resize_size, self.mean, self.std, self.interpolation, self.antialias)
        return orig_preset_forward(self, img)

    tv_presets.ImageClassification.forward = preset_forward

    # ---- resize ----
    registry = tv_utils._KERNEL_REGISTRY[tv_geo.resize]
    saved = dict(registry)
    orig_image = tv_geo.resize_image

    @functools.wraps(orig_image)
    def resize_image(image, size, interpolation=tv_geo.InterpolationMode.BILINEAR, max_size=None, antialias=True):
        if isinstance(image, torch.Tensor) and _tf.supports(image, interpolation):
            return _tf.resize_image(image, size, interpolation=interpolation, max_size=max_size, antialias=antialias)
        return orig_image(image, size, interpolation=interpolation, max_size=max_size, antialias=antialias)

    def resize_video(video, size, interpolation=tv_geo.InterpolationMode.BILINEAR, max_size=None, antialias=True):
        return resize_image(video, size, interpolation=interpolation, max_size=max_size, antialias=antialias)

    registry[torch.Tensor] = resize_image
    registry[tv_tensors.Image] = tv_utils._kernel_tv_tensor_wrapper(resize_image)
    registry[tv_tensors.Video] = tv_utils._kernel_tv_tensor_wrapper(resize_video)

    _state.update(dict(tv_boxes=tv_boxes, torchvision=torchvision, orig_batched_nms=orig_batched_nms,
                       registry=registry, saved_registry=saved, tv_poolers=tv_poolers, orig_msra=orig_msra,
                       tv_roi_align_mod=tv_roi_align_mod, orig_det_roi_align=orig_det_roi_align,
                       tv_roi_heads=tv_roi_heads, tv_rpn=tv_rpn, orig_pp=orig_pp, orig_fp=orig_fp, orig_kri=orig_kri, orig_h2k=orig_h2k,
                       tv_presets=tv_presets, orig_preset_forward=orig_preset_forward, single_stage=single_stage, matching=matching, losses=losses,
                       fcos_losses=fcos_losses, orig_mask_loss=orig_mask_loss, rcnn_transform=rcnn_transform, orig_tf_forward=orig_tf_forward, orig_tf_post=orig_tf_post))


def uninstall() -> None:
    if not _state:
        return
    torch.ops.vision_b200._install(False)
    _state["tv_boxes"].batched_nms = _state["orig_batched_nms"]
    _state["torchvision"].ops.batched_nms = _state["orig_batched_nms"]
    _state["tv_poolers"]._multiscale_roi_align = _state["orig_msra"]
    _state["tv_roi_align_mod"]._roi_align = _state["orig_det_roi_align"]
    _state["tv_presets"].ImageClassification.forward = _state["orig_preset_forward"]
    _state["tv_roi_heads"].RoIHeads.postprocess_detections = _state["orig_pp"]
    _state["tv_rpn"].RegionProposalNetwork.filter_proposals = _state["orig_fp"]
    _state["tv_roi_heads"].keypointrcnn_inference = _state["orig_kri"]
    _state["tv_roi_heads"].heatmaps_to_keypoints = _state["orig_h2k"]
    _state["tv_roi_heads"].maskrcnn_loss = _state["orig_mask_loss"]
    _state["rcnn_transform"].forward = _state["orig_tf_forward"]
    _state["rcnn_transform"].postprocess = _state["orig_tf_post"]
    for cls, orig in _state["single_stage"].items():
        cls.postprocess_detections = orig
    for (cls, name), orig in list(_state["matching"].items()) + list(_state["losses"].items()) + list(_state["fcos_losses"].items()):
        setattr(cls, name, orig)
    reg = _state["registry"]
    reg.clear()
    reg.update(_state["saved_registry"])
    _state.clear()
