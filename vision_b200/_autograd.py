"""Autograd formulas and fake (meta) kernels of the ``vision_b200::`` ops.

The reference registers these next to its kernels (torchvision/_meta_registrations.py,
torchvision/_autograd_registrations.py:340-361 in the tree; C++ Autograd keys in the 0.26 wheel).  The ``torchvision::``
ops keep the reference's registrations after install() - only their CUDA kernels (forward AND ``_*_backward``) are
replaced - so this module only concerns direct users of ``vision_b200.ops``: without it a ``requires_grad`` input would
silently produce a non-differentiable output.
"""
from __future__ import annotations

import torch

_done = False


def register() -> None:
    global _done
    if _done:
        return
    _done = True
    lib = torch.library
    ops = torch.ops.vision_b200

    # ---- roi_align ----
    def roi_align_setup(ctx, inputs, output):
        inp, rois, scale, ph, pw, sr, aligned = inputs
        ctx.save_for_backward(rois)
        ctx.in_shape = tuple(inp.shape)
        ctx.args = (scale, ph, pw, sr, aligned)

    def roi_align_backward(ctx, grad):
        (rois,) = ctx.saved_tensors
        scale, ph, pw, sr, aligned = ctx.args
        b, c, h, w = ctx.in_shape
        gi = ops._roi_align_backward(grad, rois, scale, ph, pw, b, c, h, w, sr, aligned)
        return gi, None, None, None, None, None, None

    lib.register_autograd("vision_b200::roi_align", roi_align_backward, setup_context=roi_align_setup)

    @lib.register_fake("vision_b200::roi_align")
    def _(inp, rois, spatial_scale, pooled_height, pooled_width, sampling_ratio, aligned):
        torch._check(rois.size(1) == 5, lambda: "rois must have shape as Tensor[K, 5]")
        torch._check(inp.dtype == rois.dtype, lambda: "Expected tensor for input to have the same type as tensor for rois")
        return inp.new_empty((rois.size(0), inp.size(1), pooled_height, pooled_width))

    @lib.register_fake("vision_b200::_roi_align_backward")
    def _(grad, rois, spatial_scale, pooled_height, pooled_width, batch_size, channels, height, width, sampling_ratio, aligned):
        return grad.new_empty((batch_size, channels, height, width))

    # ---- roi_pool ----
    def roi_pool_setup(ctx, inputs, output):
        inp, rois, scale, ph, pw = inputs
        ctx.save_for_backward(rois, output[1])
        ctx.mark_non_differentiable(output[1])
        ctx.in_shape = tuple(inp.shape)
        ctx.args = (scale, ph, pw)

    def roi_pool_backward(ctx, grad, _grad_argmax):
        rois, argmax = ctx.saved_tensors
        scale, ph, pw = ctx.args
        b, c, h, w = ctx.in_shape
        gi = ops._roi_pool_backward(grad, rois, argmax, scale, ph, pw, b, c, h, w)
        return gi, None, None, None, None

    lib.register_autograd("vision_b200::roi_pool", roi_pool_backward, setup_context=roi_pool_setup)

    @lib.register_fake("vision_b200::roi_pool")
    def _(inp, rois, spatial_scale, pooled_height, pooled_width):
        shape = (rois.size(0), inp.size(1), pooled_height, pooled_width)
        return inp.new_empty(shape), inp.new_empty(shape, dtype=torch.int32)

    @lib.register_fake("vision_b200::_roi_pool_backward")
    def _(grad, rois, argmax, spatial_scale, pooled_height, pooled_width, batch_size, channels, height, width):
        return grad.new_empty((batch_size, channels, height, width))

    # ---- ps_roi_align ----
    def ps_roi_align_setup(ctx, inputs, output):
        inp, rois, scale, ph, pw, sr = inputs
        ctx.save_for_backward(rois, output[1])
        ctx.mark_non_differentiable(output[1])
        ctx.in_shape = tuple(inp.shape)
        ctx.args = (scale, ph, pw, sr)

    def ps_roi_align_backward(ctx, grad, _grad_mapping):
        rois, mapping = ctx.saved_tensors
        scale, ph, pw, sr = ctx.args
        b, c, h, w = ctx.in_shape
        gi = ops._ps_roi_align_backward(grad, rois, mapping, scale, ph, pw, sr, b, c, h, w)
        return gi, None, None, None, None, None

    lib.register_autograd("vision_b200::ps_roi_align", ps_roi_align_backward, setup_context=ps_roi_align_setup)

    @lib.register_fake("vision_b200::ps_roi_align")
    def _(inp, rois, spatial_scale, pooled_height, pooled_width, sampling_ratio):
        torch._check(inp.size(1) % (pooled_height * pooled_width) == 0,
                     lambda: "input channels must be a multiple of pooling height * pooling width")
        shape = (rois.size(0), inp.size(1) // (pooled_height * pooled_width), pooled_height, pooled_width)
        return inp.new_empty(shape), inp.new_empty(shape, dtype=torch.int32)

    @lib.register_fake("vision_b200::_ps_roi_align_backward")
    def _(grad, rois, channel_mapping, spatial_scale, pooled_height, pooled_width, sampling_ratio, batch_size, channels, height,
          width):
        return grad.new_empty((batch_size, channels, height, width))

    # ---- ps_roi_pool ----
    def ps_roi_pool_setup(ctx, inputs, output):
        inp, rois, scale, ph, pw = inputs
        ctx.save_for_backward(rois, output[1])
        ctx.mark_non_differentiable(output[1])
        ctx.in_shape = tuple(inp.shape)
        ctx.args = (scale, ph, pw)

    def ps_roi_pool_backward(ctx, grad, _grad_mapping):
        rois, mapping = ctx.saved_tensors
        scale, ph, pw = ctx.args
        b, c, h, w = ctx.in_shape
        return ops._ps_roi_pool_backward(grad, rois, mapping, scale, ph, pw, b, c, h, w), None, None, None, None

    lib.register_autograd("vision_b200::ps_roi_pool", ps_roi_pool_backward, setup_context=ps_roi_pool_setup)

    @lib.register_fake("vision_b200::ps_roi_pool")
    def _(inp, rois, spatial_scale, pooled_height, pooled_width):
        shape = (rois.size(0), inp.size(1) // (pooled_height * pooled_width), pooled_height, pooled_width)
        return inp.new_empty(shape), inp.new_empty(shape, dtype=torch.int32)

    @lib.register_fake("vision_b200::_ps_roi_pool_backward")
    def _(grad, rois, channel_mapping, spatial_scale, pooled_height, pooled_width, batch_size, channels, height, width):
        return grad.new_empty((batch_size, channels, height, width))

    # ---- fused MultiScaleRoIAlign: gradients per level through _roi_align_backward on that level's RoIs ----
    def ms_setup(ctx, inputs, output):
        feats, rois, scales, ph, pw, sr = inputs[:6]
        ctx.save_for_backward(rois, output[1])
        ctx.mark_non_differentiable(output[1])
        ctx.shapes = [tuple(f.shape) for f in feats]
        ctx.args = (list(scales), ph, pw, sr)

    def ms_backward(ctx, grad, _grad_levels):
        rois, levels = ctx.saved_tensors
        scales, ph, pw, sr = ctx.args
        grads = []
        for lvl, (b, c, h, w) in enumerate(ctx.shapes):
            idx = torch.where(levels == lvl)[0]
            grads.append(ops._roi_align_backward(grad[idx].contiguous(), rois[idx].contiguous(), scales[lvl], ph, pw, b, c, h, w, sr, False))
        return (grads,) + (None,) * 10

    lib.register_autograd("vision_b200::multiscale_roi_align", ms_backward, setup_context=ms_setup)

    @lib.register_fake("vision_b200::multiscale_roi_align")
    def _(features, rois, scales, pooled_height, pooled_width, sampling_ratio, k_min, k_max, canonical_scale, canonical_level, eps):
        f0 = features[0]
        return (f0.new_empty((rois.size(0), f0.size(1), pooled_height, pooled_width)), f0.new_empty((rois.size(0),), dtype=torch.int32))

    # ---- nms / batched_nms: data-dependent output length ----
    @lib.register_fake("vision_b200::nms")
    def _(dets, scores, iou_threshold):
        ctx = torch.library.get_ctx()
        n = ctx.new_dynamic_size()
        return dets.new_empty((n,), dtype=torch.int64)

    @lib.register_fake("vision_b200::batched_nms")
    def _(boxes, scores, idxs, iou_threshold):
        ctx = torch.library.get_ctx()
        n = ctx.new_dynamic_size()
        return boxes.new_empty((n,), dtype=torch.int64)

    @lib.register_fake("vision_b200::box_iou_rotated")
    def _(boxes1, boxes2):
        return boxes1.new_empty((boxes1.size(0), boxes2.size(0)))

    # ---- resize ----
    @lib.register_fake("vision_b200::resize")
    def _(inp, out_h, out_w, mode, antialias):
        return inp.new_empty(tuple(inp.shape[:-2]) + (out_h, out_w))

    @lib.register_fake("vision_b200::rcnn_batch_images")
    def _(images, out_h, out_w, pad_h, pad_w, mean, std):
        return images[0].new_empty((len(images), images[0].shape[0], pad_h, pad_w))

    @lib.register_fake("vision_b200::match_boxes")
    def _(gt_boxes, predictions, gt_labels, high_threshold, low_threshold, allow_low_quality_matches, mode):
        n = [p.shape[0] for p in predictions]
        if mode == 1:          # VB200_MATCH_RPN: fp32 labels, matched boxes of the gt dtype (fp32 zeros without gt)
            return ([p.new_empty((k,), dtype=torch.float32) for p, k in zip(predictions, n)],
                    [p.new_empty((k, 4), dtype=g.dtype if g.numel() else torch.float32) for p, g, k in zip(predictions, gt_boxes, n)])
        out0 = [p.new_empty((k,), dtype=torch.int64) for p, k in zip(predictions, n)]
        return out0, ([p.new_empty((k,), dtype=torch.int64) for p, k in zip(predictions, n)] if mode == 2 else [])

    @lib.register_fake("vision_b200::fcos_match")
    def _(gt_boxes, anchors, radius, first_level, last_level):
        return [a.new_empty((a.shape[0],), dtype=torch.int64) for a in anchors]

    # ---- RetinaNet head losses: cls_logits and bbox_regression are the only differentiable inputs; the counts are not ----
    def cls_loss_setup(ctx, inputs, output):
        logits, matched, labels = inputs
        ctx.mark_non_differentiable(output[1])
        ctx.save_for_backward(logits, output[1])
        ctx.lists = (list(matched), list(labels))

    def cls_loss_backward(ctx, grad, _grad_counts):
        logits, counts = ctx.saved_tensors
        matched, labels = ctx.lists
        return ops.retinanet_cls_loss_backward(grad, logits, matched, labels, counts), [None] * len(matched), [None] * len(labels)

    lib.register_autograd("vision_b200::retinanet_cls_loss", cls_loss_backward, setup_context=cls_loss_setup)

    def box_loss_setup(ctx, inputs, output):
        regression, anchors, gt_boxes, matched, weights = inputs
        ctx.mark_non_differentiable(output[1])
        ctx.save_for_backward(regression, output[1])
        ctx.lists = (list(anchors), list(gt_boxes), list(matched), list(weights))

    def box_loss_backward(ctx, grad, _grad_counts):
        regression, counts = ctx.saved_tensors
        anchors, gt_boxes, matched, weights = ctx.lists
        return (ops.retinanet_box_loss_backward(grad, regression, anchors, gt_boxes, matched, weights, counts), [None] * len(anchors),
                [None] * len(gt_boxes), [None] * len(matched), None)

    lib.register_autograd("vision_b200::retinanet_box_loss", box_loss_backward, setup_context=box_loss_setup)

    @lib.register_fake("vision_b200::retinanet_cls_loss")
    def _(cls_logits, matched_idxs, labels):
        return cls_logits.new_empty(()), cls_logits.new_empty((cls_logits.shape[0],), dtype=torch.int64)

    @lib.register_fake("vision_b200::retinanet_cls_loss_backward")
    def _(grad, cls_logits, matched_idxs, labels, num_foreground):
        return cls_logits.new_empty(cls_logits.shape)

    @lib.register_fake("vision_b200::retinanet_box_loss")
    def _(bbox_regression, anchors, gt_boxes, matched_idxs, weights):
        return bbox_regression.new_empty(()), bbox_regression.new_empty((bbox_regression.shape[0],), dtype=torch.int64)

    @lib.register_fake("vision_b200::retinanet_box_loss_backward")
    def _(grad, bbox_regression, anchors, gt_boxes, matched_idxs, weights, num_foreground):
        return bbox_regression.new_empty(bbox_regression.shape)

    # ---- deform_conv2d ----
    def dcn_setup(ctx, inputs, output):
        inp, weight, offset, mask, bias = inputs[:5]
        ctx.save_for_backward(inp, weight, offset, mask, bias)
        ctx.args = tuple(inputs[5:])

    def dcn_backward(ctx, grad):
        inp, weight, offset, mask, bias = ctx.saved_tensors
        gi, gw, go, gm, gb = ops._deform_conv2d_backward(grad, inp, weight, offset, mask, bias, *ctx.args)
        return (gi, gw, go, gm, gb) + (None,) * 9

    lib.register_autograd("vision_b200::deform_conv2d", dcn_backward, setup_context=dcn_setup)

    @lib.register_fake("vision_b200::_deform_conv2d_backward")
    def _(grad, inp, weight, offset, mask, bias, *args):
        return (torch.empty_like(inp), torch.empty_like(weight), torch.empty_like(offset), torch.empty_like(mask), torch.empty_like(bias))

    @lib.register_fake("vision_b200::deform_conv2d")
    def _(inp, weight, offset, mask, bias, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, groups, offset_groups, use_mask):
        kh, kw = weight.shape[-2:]
        out_h = (inp.shape[2] + 2 * pad_h - (dil_h * (kh - 1) + 1)) // stride_h + 1
        out_w = (inp.shape[3] + 2 * pad_w - (dil_w * (kw - 1) + 1)) // stride_w + 1
        return inp.new_empty((inp.shape[0], weight.shape[0], out_h, out_w))
