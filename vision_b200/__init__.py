"""vision_b200 — Hopper-native (sm_90a) kernels behind torchvision's custom-op hot path.

    import torchvision, vision_b200
    vision_b200.install()        # torchvision.ops.{nms, roi_align, roi_pool, ps_roi_align, deform_conv2d}
                                 # on CUDA tensors, torchvision.ops.batched_nms and
                                 # transforms.v2.functional.resize now run the kernels in this package
    vision_b200.uninstall()      # reference kernels are active again

The same ops are callable directly as ``vision_b200.ops.*`` / ``vision_b200.transforms.*``.
"""
from __future__ import annotations

from . import _lib, detection, ops, transforms  # noqa: F401
from ._install import install, installed, uninstall  # noqa: F401

__all__ = ["ops", "transforms", "install", "uninstall", "installed", "launch_count", "set_nms_semantics"]


def launch_count() -> int:
    """Kernel launches issued by libvision_b200 so far in this process."""
    return int(_lib.core().vb200_launch_count())


def set_nms_semantics(which: str) -> None:
    """'cuda' (default): IoU arithmetic of the compiled reference CUDA kernel; 'cpu': of the CPU kernel."""
    import torch

    _lib.load_ops()
    torch.ops.vision_b200._set_nms_semantics({"cpu": 0, "cuda": 1}[which])
