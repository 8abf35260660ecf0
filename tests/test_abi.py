"""CPU suite, part 2: the C-ABI library loads and exports every symbol include/vision_b200.h
declares (no compute calls without a GPU), and install() leaves the CPU path alone (cfg1 plumbing)."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    text = open(os.path.join(ROOT, "include", "vision_b200.h")).read()
    return sorted(set(re.findall(r"^VB200_API [\w\s\*]+?\b(vb200_\w+)\(", text, flags=re.M)))


def test_header_symbols_exported_at_abi_version_2():
    from vision_b200 import _lib

    lib = _lib.core()
    declared = _declared()
    assert len(declared) >= 14
    assert sorted(_lib.ABI_SYMBOLS) == declared
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/vision_b200.h but not exported"
    assert lib.vb200_abi_version() == 2


def test_header_cites_reference_for_each_entry_point():
    text = open(os.path.join(ROOT, "include", "vision_b200.h")).read()
    for op in ("roi_align_kernel.cu", "roi_pool_kernel.cu", "ps_roi_align_kernel.cu", "nms_kernel.cu",
               "deform_conv2d_kernel.cu", "boxes.py", "_geometry.py"):
        assert op in text


def test_workspace_queries_need_no_gpu():
    from vision_b200 import _lib
    import ctypes

    lib = _lib.core()
    assert lib.vb200_nms_workspace_bytes(ctypes.c_int64(0)) == 0
    assert lib.vb200_nms_workspace_bytes(ctypes.c_int64(1000)) > 1000 * 20
    assert lib.vb200_batched_nms_workspace_bytes(ctypes.c_int64(100000)) > 100000 * 60


def test_batched_nms_workspace_stays_small():
    """A 100k-box batched_nms takes the fused per-class path; its workspace must not carry the n x n/64-bit matrix of
    the plain-nms pipeline (1.25 GB at this size), only the 33-words-per-row class mask (26 MB) and the sort buffers."""
    from vision_b200 import _lib
    import ctypes

    lib = _lib.core()
    lib.vb200_batched_nms_workspace_bytes.restype = ctypes.c_size_t
    lib.vb200_nms_workspace_bytes.restype = ctypes.c_size_t
    assert lib.vb200_batched_nms_workspace_bytes(ctypes.c_int64(100_000)) < 64 << 20
    # inside the reference's coordinate-trick range the plain-nms matrix is part of it (and small)
    assert lib.vb200_batched_nms_workspace_bytes(ctypes.c_int64(25_000)) < 128 << 20
    assert lib.vb200_nms_workspace_bytes(ctypes.c_int64(1000)) < 1 << 20


def test_missing_extension_fails_loudly(monkeypatch, tmp_path):
    from vision_b200 import _lib

    monkeypatch.setattr(_lib, "_core", None)
    monkeypatch.setattr(_lib, "CORE_LIB", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.ExtensionMissing):
        _lib.core()


def test_ops_refuse_cpu_tensors():
    import torch
    import vision_b200

    with pytest.raises(RuntimeError, match="no CPU path"):
        vision_b200.ops.nms(torch.zeros(2, 4), torch.zeros(2), 0.5)
    with pytest.raises(RuntimeError, match="no CPU path"):
        vision_b200.transforms.resize_image(torch.zeros(3, 8, 8), [4, 4])


def test_cfg1_plumbing_cpu_nms_unchanged(golden):
    """BASELINE configs[0]: torchvision.ops.nms on 1000 CPU boxes with our package installed must still
    hit the reference CPU kernel and return identical indices."""
    tv = pytest.importorskip("torchvision")
    import torch
    import vision_b200

    b, s = torch.from_numpy(golden["cfg1_boxes"]), torch.from_numpy(golden["cfg1_scores"])
    before = tv.ops.nms(b, s, 0.5)
    vision_b200.install()
    try:
        assert vision_b200.installed()
        after = tv.ops.nms(b, s, 0.5)
        idx = torch.randint(0, 4, (1000,))
        bn = tv.ops.batched_nms(b, s, idx, 0.5)
        from torchvision.transforms.v2 import functional as F

        img = torch.rand(3, 17, 11)
        rz = F.resize(img, [12, 13])
        dump = torch._C._dispatch_dump("torchvision::roi_align")
        assert "torch_shim.cpp" in [l for l in dump.split("\n") if l.startswith("CUDA:")][0]
    finally:
        vision_b200.uninstall()
    assert torch.equal(before, after) and np.array_equal(after.numpy(), golden["cfg1_keep"])
    assert torch.equal(bn, tv.ops.batched_nms(b, s, idx, 0.5))
    assert torch.equal(rz, F.resize(img, [12, 13]))
    dump = torch._C._dispatch_dump("torchvision::roi_align")
    assert "torch_shim.cpp" not in [l for l in dump.split("\n") if l.startswith("CUDA:")][0]
