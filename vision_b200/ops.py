"""Host-side mirror of ``torchvision.ops`` for the hot path: same names, arguments and errors
(torchvision/ops/boxes.py:20-126, roi_align.py:204-285, roi_pool.py:15-53, ps_roi_align.py:11-59,
deform_conv.py:14-107), routed to the sm_90a kernels through ``torch.ops.vision_b200``.

These functions accept CUDA tensors only — there is no CPU path in this package (the reference's
CPU kernels keep serving CPU tensors through ``torchvision.ops`` itself, untouched by install()).
"""
from __future__ import annotations

import torch
from torch import Tensor
from torch.nn.modules.utils import _pair

from . import _lib


def _ops():
    _lib.load_ops()
    return torch.ops.vision_b200


def _require_cuda(t: Tensor, name: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(
            f"vision_b200.ops: `{name}` must be a CUDA tensor (got {t.device}); this package has no CPU path — "
            f"use torchvision.ops for CPU tensors"
        )


# ---- boxes ------------------------------------------------------------------
def nms(boxes: Tensor, scores: Tensor, iou_threshold: float) -> Tensor:
    """torchvision.ops.nms (boxes.py:20-54): int64 indices of kept boxes, descending score."""
    _require_cuda(boxes, "boxes")
    return _ops().nms(boxes, scores, float(iou_threshold))


def batched_nms(boxes: Tensor, scores: Tensor, idxs: Tensor, iou_threshold: float) -> Tensor:
    """torchvision.ops.batched_nms (boxes.py:57-89) as ONE fused device pipeline.

    Same strategy switch as the reference for CUDA tensors (boxes.py:86): numel > 100_000 ->
    per-class ("vanilla") semantics on un-offset coordinates, else the coordinate trick."""
    _require_cuda(boxes, "boxes")
    return _ops().batched_nms(boxes, scores, idxs, float(iou_threshold))


def box_iou_rotated(boxes1: Tensor, boxes2: Tensor) -> Tensor:
    """IoU of rotated boxes in cxcywhr format (torchvision.ops.box_iou(..., fmt="cxcywhr") -> torch.ops.torchvision.box_iou_rotated,
    torchvision/ops/boxes.py:386-399).  The installed 0.26 wheel has no such op, so this is only reachable as vision_b200.ops."""
    _require_cuda(boxes1, "boxes1")
    return _ops().box_iou_rotated(boxes1, boxes2)


# ---- RoI ops ------------------------------------------------------------------
# box-list handling and its assertion texts are the reference's own helpers (torchvision/ops/_utils.py:18-38), not re-typed
from torchvision.ops._utils import check_roi_boxes_shape, convert_boxes_to_roi_format  # noqa: E402,F401


def _rois(boxes) -> Tensor:
    check_roi_boxes_shape(boxes)
    return boxes if isinstance(boxes, torch.Tensor) else convert_boxes_to_roi_format(boxes)


def roi_align(input: Tensor, boxes, output_size, spatial_scale: float = 1.0, sampling_ratio: int = -1,
              aligned: bool = False) -> Tensor:
    """torchvision.ops.roi_align (roi_align.py:204-285)."""
    _require_cuda(input, "input")
    rois = _rois(boxes)
    output_size = _pair(output_size)
    return _ops().roi_align(input, rois, float(spatial_scale), output_size[0], output_size[1], int(sampling_ratio),
                            bool(aligned))


def roi_pool(input: Tensor, boxes, output_size, spatial_scale: float = 1.0) -> Tensor:
    """torchvision.ops.roi_pool (roi_pool.py:15-53); the argmax tensor is dropped as in the reference."""
    _require_cuda(input, "input")
    rois = _rois(boxes)
    output_size = _pair(output_size)
    output, _ = _ops().roi_pool(input, rois, float(spatial_scale), output_size[0], output_size[1])
    return output


def ps_roi_align(input: Tensor, boxes, output_size, spatial_scale: float = 1.0, sampling_ratio: int = -1) -> Tensor:
    """torchvision.ops.ps_roi_align (ps_roi_align.py:11-59)."""
    _require_cuda(input, "input")
    rois = _rois(boxes)
    output_size = _pair(output_size)
    output, _ = _ops().ps_roi_align(input, rois, float(spatial_scale), output_size[0], output_size[1],
                                    int(sampling_ratio))
    return output


def ps_roi_pool(input: Tensor, boxes, output_size, spatial_scale: float = 1.0) -> Tensor:
    """torchvision.ops.ps_roi_pool (ps_roi_pool.py:11-52)."""
    _require_cuda(input, "input")
    rois = _rois(boxes)
    output_size = _pair(output_size)
    output, _ = _ops().ps_roi_pool(input, rois, float(spatial_scale), output_size[0], output_size[1])
    return output


# ---- deform_conv2d --------------------------------------------------------------
def deform_conv2d(input: Tensor, offset: Tensor, weight: Tensor, bias=None, stride=(1, 1), padding=(0, 0),
                  dilation=(1, 1), mask=None) -> Tensor:
    """torchvision.ops.deform_conv2d (deform_conv.py:14-107), incl. the dummy mask/bias convention."""
    _require_cuda(input, "input")
    out_channels = weight.shape[0]
    use_mask = mask is not None
    if mask is None:
        mask = torch.zeros((input.shape[0], 1), device=input.device, dtype=input.dtype)
    if bias is None:
        bias = torch.zeros(out_channels, device=input.device, dtype=input.dtype)
    stride_h, stride_w = _pair(stride)
    pad_h, pad_w = _pair(padding)
    dil_h, dil_w = _pair(dilation)
    weights_h, weights_w = weight.shape[-2:]
    _, n_in_channels, _, _ = input.shape
    n_offset_grps = offset.shape[1] // (2 * weights_h * weights_w)
    n_weight_grps = n_in_channels // weight.shape[1]
    if n_offset_grps == 0:
        raise RuntimeError(
            "the shape of the offset tensor at dimension 1 is not valid. It should "
            "be a multiple of 2 * weight.size[2] * weight.size[3].\n"
            f"Got offset.shape[1]={offset.shape[1]}, while 2 * weight.size[2] * weight.size[3]={2 * weights_h * weights_w}"
        )
    return _ops().deform_conv2d(input, weight, offset, mask, bias, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w,
                                n_weight_grps, n_offset_grps, use_mask)


# ---- MultiScaleRoIAlign ------------------------------------------------------------
def multiscale_roi_align_supported(x_filtered, boxes, output_size, sampling_ratio) -> bool:
    """True when the fused kernel covers the call (else torchvision's per-level loop runs, each level on our roi_align)."""
    if len(x_filtered) < 2 or len(x_filtered) > 8 or tuple(output_size) != (7, 7) or int(sampling_ratio) != 2:
        return False
    f0 = x_filtered[0]
    if not all(isinstance(f, Tensor) and f.is_cuda and f.dtype == torch.float32 and f.dim() == 4 and f.shape[:2] == f0.shape[:2]
               for f in x_filtered):
        return False
    if not all(isinstance(b, Tensor) and b.is_cuda and b.dtype == torch.float32 for b in boxes):
        return False
    import ctypes

    n = len(x_filtered)
    hs = (ctypes.c_int * n)(*[int(f.shape[2]) for f in x_filtered])
    ws = (ctypes.c_int * n)(*[int(f.shape[3]) for f in x_filtered])
    return bool(_lib.core().vb200_multiscale_roi_align_supported(0, n, hs, ws, 7, 7, 2))


def multiscale_roi_align(x_filtered, boxes, output_size, sampling_ratio, scales, mapper) -> Tensor:
    """_multiscale_roi_align (torchvision/ops/poolers.py:147-228) as ONE fused call: the LevelMapper (poolers.py:47-84) is
    evaluated on the device, every level is pooled by the same launch and rows are written in place."""
    if scales is None or mapper is None:
        raise ValueError("scales and mapper should not be None")
    rois = convert_boxes_to_roi_format(list(boxes))
    out, _levels = _ops().multiscale_roi_align(list(x_filtered), rois, [float(s) for s in scales], int(output_size[0]),
                                               int(output_size[1]), int(sampling_ratio), int(mapper.k_min), int(mapper.k_max),
                                               float(mapper.s0), float(mapper.lvl0), float(mapper.eps))
    return out
