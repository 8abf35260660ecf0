"""Loading of the native libraries.  There is no CPU / eager fallback: if the CUDA extension is
missing the import of any op fails loudly (RuntimeError), as the tier contract requires."""
from __future__ import annotations

import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_DIR = os.path.join(_HERE, "lib")
CORE_LIB = os.path.join(LIB_DIR, "libvision_b200.so")
SHIM_LIB = os.path.join(LIB_DIR, "libvision_b200_torch.so")

_lock = threading.Lock()
_core = None
_shim_loaded = False


class ExtensionMissing(RuntimeError):
    pass


def _missing(path: str) -> ExtensionMissing:
    return ExtensionMissing(
        f"vision_b200 native library not found: {path}. Build it in-tree with "
        f"`python -m vision_b200.build` (needs nvcc, -gencode arch=compute_90a,code=sm_90a). "
        f"There is deliberately no CPU fallback."
    )


def core() -> ctypes.CDLL:
    """The C-ABI kernel library (include/vision_b200.h) through ctypes."""
    global _core
    with _lock:
        if _core is None:
            if not os.path.exists(CORE_LIB):
                raise _missing(CORE_LIB)
            lib = ctypes.CDLL(CORE_LIB, mode=ctypes.RTLD_GLOBAL)
            lib.vb200_last_error.restype = ctypes.c_char_p
            lib.vb200_launch_count.restype = ctypes.c_uint64
            lib.vb200_reload_env.restype = None
            for name in ("vb200_nms_workspace_bytes", "vb200_batched_nms_workspace_bytes",
                         "vb200_roi_align_workspace_bytes", "vb200_deform_conv2d_workspace_bytes",
                         "vb200_roi_backward_workspace_bytes", "vb200_multiscale_roi_align_workspace_bytes",
                         "vb200_detection_postprocess_workspace_bytes", "vb200_deform_conv2d_packed_weight_bytes",
                         "vb200_single_stage_postprocess_workspace_bytes",
                         "vb200_deform_conv2d_backward_inputs_workspace_bytes", "vb200_heatmaps_to_keypoints_workspace_bytes",
                         "vb200_match_boxes_workspace_bytes"):
                getattr(lib, name).restype = ctypes.c_size_t
            _core = lib
        return _core


def load_ops() -> None:
    """Loads the torch dispatcher shim: defines torch.ops.vision_b200.*"""
    global _shim_loaded
    with _lock:
        if _shim_loaded:
            return
        for p in (CORE_LIB, SHIM_LIB):
            if not os.path.exists(p):
                raise _missing(p)
        import torch

        torch.ops.load_library(SHIM_LIB)
        _shim_loaded = True
    from . import _autograd

    _autograd.register()      # autograd formulas + fake kernels of the vision_b200:: ops


# every symbol include/vision_b200.h declares (checked by tests/test_abi.py)
ABI_SYMBOLS = (
    "vb200_abi_version", "vb200_last_error", "vb200_launch_count", "vb200_reload_env",
    "vb200_roi_align_workspace_bytes", "vb200_roi_align_forward", "vb200_roi_align_forward_gather", "vb200_roi_pool_forward",
    "vb200_ps_roi_align_forward", "vb200_nms_workspace_bytes", "vb200_nms",
    "vb200_batched_nms_workspace_bytes", "vb200_batched_nms", "vb200_deform_conv2d_workspace_bytes",
    "vb200_deform_conv2d_forward", "vb200_resize", "vb200_resize_gather",
    "vb200_deform_conv2d_packed_weight_bytes", "vb200_deform_conv2d_pack_weight",
    "vb200_deform_conv2d_sample_columns", "vb200_deform_conv2d_backward_inputs", "vb200_ps_roi_pool_forward", "vb200_ps_roi_pool_backward", "vb200_box_iou_rotated", "vb200_resize_crop_normalize", "vb200_detection_postprocess_workspace_bytes", "vb200_detection_postprocess",
    "vb200_multiscale_roi_align_workspace_bytes", "vb200_multiscale_roi_align_supported", "vb200_multiscale_roi_align_forward",
    "vb200_roi_backward_workspace_bytes", "vb200_roi_align_backward", "vb200_roi_pool_backward", "vb200_ps_roi_align_backward",
    "vb200_single_stage_postprocess_workspace_bytes", "vb200_single_stage_postprocess",
    "vb200_deform_conv2d_backward_inputs_workspace_bytes", "vb200_roi_backward_deterministic_supported",
    "vb200_heatmaps_to_keypoints_workspace_bytes", "vb200_heatmaps_to_keypoints",
    "vb200_rcnn_batch_images", "vb200_rcnn_rescale", "vb200_match_boxes_workspace_bytes", "vb200_match_boxes",
    "vb200_fcos_level_bounds", "vb200_fcos_match", "vb200_head_loss_workspace_bytes", "vb200_head_loss", "vb200_head_loss_backward",
    "vb200_mask_loss_workspace_bytes", "vb200_mask_loss", "vb200_mask_loss_backward",
)
