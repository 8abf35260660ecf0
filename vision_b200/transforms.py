"""Host-side mirror of ``torchvision.transforms.v2.functional.resize`` for tensors
(torchvision/transforms/v2/functional/_geometry.py:236-362, transforms/functional.py:353-384).

Output-size rules, interpolation checks and the "same size -> return input" shortcut are the
reference's; the compute is ONE fused sm_90a kernel (storage dtype in, fp32 math, storage dtype
out) instead of cast -> aten::upsample_* -> cast.
"""
from __future__ import annotations

from enum import Enum
from typing import Optional, Sequence, Union

import torch

from . import _lib


class InterpolationMode(Enum):
    """Values match torchvision.transforms.InterpolationMode (transforms/functional.py:23-36)."""
    NEAREST = "nearest"
    NEAREST_EXACT = "nearest-exact"
    BILINEAR = "bilinear"
    BICUBIC = "bicubic"
    BOX = "box"
    HAMMING = "hamming"
    LANCZOS = "lanczos"


_PIL_INT_TO_MODE = {0: "nearest", 2: "bilinear", 3: "bicubic", 4: "box", 5: "hamming", 1: "lanczos"}
_FUSED_DTYPES = (torch.float32, torch.float16, torch.bfloat16, torch.uint8)
_MODE_CODE = {"bilinear": 0, "bicubic": 1}


def _mode_value(interpolation) -> str:
    """_check_interpolation (_geometry.py:36-51), tolerant of torchvision's own enum."""
    if isinstance(interpolation, str):
        valid = [m.value for m in InterpolationMode]
        if interpolation not in valid:
            raise ValueError(
                f"Invalid interpolation mode: '{interpolation}'. Supported string values are: {valid}."
            )
        return interpolation
    if isinstance(interpolation, bool):
        raise ValueError(f"Argument interpolation should be an `InterpolationMode`, but got {interpolation}.")
    if isinstance(interpolation, int):
        if interpolation not in _PIL_INT_TO_MODE:
            raise ValueError(f"Unknown Pillow interpolation constant {interpolation}")
        return _PIL_INT_TO_MODE[interpolation]
    value = getattr(interpolation, "value", None)
    if isinstance(interpolation, Enum) and isinstance(value, str) and value in [m.value for m in InterpolationMode]:
        return value
    raise ValueError(
        "Argument interpolation should be an `InterpolationMode` or a corresponding Pillow integer constant, "
        f"but got {interpolation}."
    )


def compute_resized_output_size(canvas_size: Sequence[int], size, max_size: Optional[int] = None) -> list[int]:
    """The reference's own rule, not a restatement: _compute_resized_output_size (_geometry.py:236-246 ->
    transforms/functional.py:353-384), incl. its ValueError texts."""
    from torchvision.transforms.v2.functional._geometry import _compute_resized_output_size

    if isinstance(size, int):
        size = [size]
    return list(_compute_resized_output_size(tuple(canvas_size), size=None if size is None else list(size), max_size=max_size))


def supports(image: torch.Tensor, interpolation) -> bool:
    """True when resize_image runs on the fused CUDA kernel (bilinear / bicubic, fp32/fp16/bf16/uint8)."""
    try:
        mode = _mode_value(interpolation)
    except ValueError:
        return False
    return image.is_cuda and mode in _MODE_CODE and image.dtype in _FUSED_DTYPES and image.dim() >= 3


def resize_image(image: torch.Tensor, size, interpolation: Union[str, InterpolationMode, int] = InterpolationMode.BILINEAR,
                 max_size: Optional[int] = None, antialias: Optional[bool] = True) -> torch.Tensor:
    """resize_image (_geometry.py:283-362) for CUDA tensors [..., C, H, W]."""
    mode = _mode_value(interpolation)
    antialias = False if antialias is None else antialias
    if mode not in _MODE_CODE:
        raise RuntimeError(
            f"vision_b200.resize_image implements bilinear and bicubic only (got '{mode}'); "
            f"other modes stay on torchvision's own kernel"
        )
    if not image.is_cuda:
        raise RuntimeError("vision_b200.resize_image needs a CUDA tensor; this package has no CPU path")
    if image.dtype not in _FUSED_DTYPES:
        raise RuntimeError(f"vision_b200.resize_image: unsupported dtype {image.dtype}")
    shape = image.shape
    num_channels, old_height, old_width = shape[-3:]
    new_height, new_width = compute_resized_output_size((old_height, old_width), size=size, max_size=max_size)
    if (new_height, new_width) == (old_height, old_width):
        return image
    if image.numel() == 0:
        return image.reshape(shape[:-3] + (num_channels, new_height, new_width))
    _lib.load_ops()
    out = torch.ops.vision_b200.resize(image.reshape(-1, num_channels, old_height, old_width), new_height, new_width,
                                       _MODE_CODE[mode], bool(antialias))
    return out.reshape(shape[:-3] + (num_channels, new_height, new_width))


def resize(inpt: torch.Tensor, size, interpolation=InterpolationMode.BILINEAR, max_size: Optional[int] = None,
           antialias: Optional[bool] = True) -> torch.Tensor:
    """transforms.v2.functional.resize (_geometry.py:249-263) for plain tensors / tv_tensors.Image/Video."""
    return resize_image(inpt, size=size, interpolation=interpolation, max_size=max_size, antialias=antialias)


# ---- fused inference preprocessing (SURVEY.md §8f4) ---------------------------------------------------------------
def classification_preprocess_supported(img, crop_size, resize_size, interpolation, antialias) -> bool:
    if not (isinstance(img, torch.Tensor) and img.is_cuda and img.dtype in _FUSED_DTYPES and img.dim() in (3, 4)):
        return False
    if img.shape[-3] > 8 or img.numel() == 0:
        return False
    try:
        mode = _mode_value(interpolation)
    except ValueError:
        return False
    if mode not in _MODE_CODE or antialias not in (True, False):
        return False
    if mode == "bicubic" and not antialias:
        return False
    h, w = img.shape[-2:]
    rh, rw = compute_resized_output_size((h, w), size=list(resize_size))
    ch, cw = _crop_hw(crop_size)
    return ch <= rh and cw <= rw and (rh, rw) != (h, w)


def _crop_hw(crop_size):
    if isinstance(crop_size, int):
        return crop_size, crop_size
    if len(crop_size) == 1:
        return int(crop_size[0]), int(crop_size[0])
    return int(crop_size[0]), int(crop_size[1])


def classification_preprocess(img: torch.Tensor, crop_size, resize_size, mean, std, interpolation=InterpolationMode.BILINEAR,
                              antialias: Optional[bool] = True) -> torch.Tensor:
    """ImageClassification.forward (torchvision/transforms/_presets.py:57-64) as ONE kernel: resize (shorter edge to
    `resize_size`) -> center_crop(`crop_size`) -> convert_image_dtype(float) -> normalize(mean, std).  CUDA tensors
    [C, H, W] or [B, C, H, W], uint8 / fp16 / bf16 / fp32; returns fp32."""
    if not classification_preprocess_supported(img, crop_size, resize_size, interpolation, antialias):
        raise RuntimeError("vision_b200.classification_preprocess: unsupported input (CUDA tensor, bilinear or bicubic+antialias, "
                           "crop inside the resized image); use torchvision's preset for the rest")
    _lib.load_ops()
    squeeze = img.dim() == 3
    x = img.unsqueeze(0) if squeeze else img
    h, w = x.shape[-2:]
    rh, rw = compute_resized_output_size((h, w), size=list(resize_size))
    ch, cw = _crop_hw(crop_size)
    top = int(round((rh - ch) / 2.0))          # transforms/functional.py center_crop
    left = int(round((rw - cw) / 2.0))
    out = torch.ops.vision_b200.resize_crop_normalize(x, rh, rw, top, left, ch, cw, _MODE_CODE[_mode_value(interpolation)], bool(antialias),
                                                      [float(m) for m in mean], [float(s) for s in std])
    return out.squeeze(0) if squeeze else out
