"""One small call of every kernel path, meant to run under compute-sanitizer (memcheck / racecheck):
    compute-sanitizer --tool memcheck python tools/sanitize_smoke.py
    compute-sanitizer --tool memcheck python tools/sanitize_smoke.py matching     (the box-matching kernels: memcheck only)
    compute-sanitizer --tool memcheck python tools/sanitize_smoke.py fcos         (the FCOS matching kernel: memcheck only)
    compute-sanitizer --tool memcheck python tools/sanitize_smoke.py retinanet_loss   (the head-loss kernels: memcheck only)
No numerics are checked here (tests/ does that); the point is out-of-bounds / hazard reports."""
import os
import sys

import torch

sys.path.insert(0, ".")
import vision_b200 as vb
from vision_b200 import workloads

dev = "cuda"
only = sys.argv[1] if len(sys.argv) > 1 else "all"


def env(k, v):
    if v is None:
        os.environ.pop(k, None)
    else:
        os.environ[k] = v
    vb._lib.core().vb200_reload_env()


def roi():
    x, r, kw = workloads.cfg2_roi_align(seed=1, k=300, batch=2, channels=16, height=40, width=52)
    r = r.clone()
    r[::7, 1:3] -= 90.0
    r[1::11, 3:] += 400.0
    x, r = x.to(dev), r.to(dev)
    for path in ("line", "plane", "generic"):
        env("VB200_ROI_ALIGN_PATH", path)
        vb.ops.roi_align(x, r, 7, 0.25, 2, False)
        vb.ops.roi_align(x, r, 7, 0.25, 2, True)
    env("VB200_ROI_ALIGN_PATH", None)
    vb.ops.roi_align(x.half(), r.half(), (3, 5), 0.25, -1, False)
    vb.ops.roi_pool(x, r, 7, 0.25)
    xp = torch.randn(2, 2 * 9, 20, 24, device=dev)
    vb.ops.ps_roi_align(xp, r[:50], 3, 0.25, 2)


def bwd():
    """roi_align / roi_pool / ps_roi_align backward, default and deterministic: atomic plane, row-owning plane (one and several
    table chunks) and generic atomic kernels; tiny RoIs (duplicate columns) and boxes outside the image"""
    vb._lib.load_ops()
    x, r, kw = workloads.cfg2_roi_align(seed=2, k=120, batch=2, channels=4, height=30, width=36)
    r = r.clone()
    r[::7, 1:3] -= 90.0
    r[1::11, 3:] += 400.0
    r[2::9, 3:] = r[2::9, 1:3] + 0.5
    x, r = x.to(dev), r.to(dev)
    xp = torch.randn(2, 2 * 9, 30, 36, device=dev)
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        for ph, pw, sr in ((7, 7, 2), (14, 14, 3), (3, 20, 2)):
            g = torch.randn(120, 4, ph, pw, device=dev)
            for aligned in (False, True):
                torch.ops.vision_b200._roi_align_backward(g, r, 0.25, ph, pw, 2, 4, 30, 36, sr, aligned)
        out, am = torch.ops.vision_b200.roi_pool(x, r, 0.25, 7, 7)
        torch.ops.vision_b200._roi_pool_backward(torch.randn_like(out), r, am, 0.25, 7, 7, 2, 4, 30, 36)
        out, cm = torch.ops.vision_b200.ps_roi_align(xp, r, 0.25, 3, 3, 2)
        torch.ops.vision_b200._ps_roi_align_backward(torch.randn_like(out), r, cm, 0.25, 3, 3, 2, 2, 18, 30, 36)
    torch.use_deterministic_algorithms(False)
    torch.ops.vision_b200._roi_align_backward(torch.randn(120, 4, 7, 7, device=dev).double(), r.double(), 0.25, 7, 7, 2, 4, 30, 36,
                                              2, False)


def nms():
    for n in (1, 300, 5000):
        b, s, i = [t.to(dev) for t in workloads.cfg3_batched_nms(n=n)]
        for path in ("mask", "chain"):
            env("VB200_NMS_PATH", path)
            vb.ops.nms(b, s, 0.5)
        env("VB200_NMS_PATH", None)
    b, s, i = [t.to(dev) for t in workloads.cfg3_batched_nms(n=30000, classes=40)]
    i[:6000] = 0
    for path in (None, "chain"):
        env("VB200_BNMS_PATH", path)
        vb.ops.batched_nms(b, s, i, 0.5)
    env("VB200_BNMS_PATH", None)
    vb.ops.batched_nms(b[:3000], s[:3000], i[:3000], 0.5)            # coordinate trick
    vb.ops.nms(b[:700].double(), s[:700].double(), 0.5)


def resize():
    for dt in (torch.float16, torch.bfloat16, torch.float32, torch.uint8):
        x = torch.rand(2, 3, 96, 1024, device=dev)
        x = (x * 255).to(torch.uint8) if dt == torch.uint8 else x.to(dt)
        for path in (None, "generic"):
            env("VB200_RESIZE_PATH", path)
            vb.transforms.resize_image(x, [17, 40], antialias=True)
        env("VB200_RESIZE_PATH", None)
        vb.transforms.resize_image(x, [17, 40], antialias=False)
        vb.transforms.resize_image(x, [120, 1100], interpolation="bicubic", antialias=True)


def dcn():
    for dt, cin, cout in ((torch.bfloat16, 64, 128), (torch.float16, 128, 512), (torch.float32, 6, 4)):
        x = torch.randn(2, cin, 12, 12, device=dev).to(dt)
        w = torch.randn(cout, cin, 3, 3, device=dev).to(dt) * 0.05
        off = torch.randn(2, 18, 12, 12, device=dev).to(dt) * 2
        m = torch.rand(2, 9, 12, 12, device=dev).to(dt)
        bias = torch.randn(cout, device=dev).to(dt)
        vb.ops.deform_conv2d(x, off, w, bias, (1, 1), (1, 1), (1, 1), m)
        vb.ops.deform_conv2d(x, off, w, None, (1, 1), (1, 1), (1, 1), None)
        env("VB200_DCN_PATH", "simt")
        vb.ops.deform_conv2d(x, off, w, bias, (1, 1), (1, 1), (1, 1), m)
        env("VB200_DCN_PATH", None)


def gather():
    """the multi-destination stores of the fused all-gather (roi_align, resize, deform_conv2d)"""
    x, r, kw = workloads.cfg2_roi_align(seed=3, k=200, batch=2, channels=8, height=80, width=200)
    r = r.clone()
    r[::7, 1:3] -= 90.0
    r[1::11, 3:] += 400.0
    x, r = x.to(dev), r.to(dev)
    want = vb.ops.roi_align(x, r, 7, 0.25, 2, False)
    bufs = [torch.empty_like(want) for _ in range(3)]
    torch.ops.vision_b200.roi_align_gather(x, r, [b.data_ptr() for b in bufs], 0, 0.25, 7, 7, 2, False)
    img = torch.rand(2, 3, 96, 1024, device=dev).half()
    o = [torch.empty(2, 3, 17, 40, device=dev, dtype=torch.float16) for _ in range(3)]
    torch.ops.vision_b200.resize_gather(img, [t.data_ptr() for t in o], 17, 40, 0, True)
    xi = torch.randn(2, 64, 12, 12, device=dev).bfloat16()
    w = (torch.randn(128, 64, 3, 3, device=dev) * 0.05).bfloat16()
    off = (torch.randn(2, 18, 12, 12, device=dev) * 2).bfloat16()
    m = torch.rand(2, 9, 12, 12, device=dev).bfloat16()
    bias = torch.randn(128, device=dev).bfloat16()
    d = [torch.empty(2, 128, 12, 12, device=dev, dtype=torch.bfloat16) for _ in range(3)]
    torch.ops.vision_b200.deform_conv2d_gather(xi, w, off, m, bias, [t.data_ptr() for t in d], 1, 1, 1, 1, 1, 1, 1, 1, True)


def matching():
    """the box-matching kernels, memcheck only: every mode, a background image, a gt count past one shared-memory chunk, a
    partial last tile, fp16 / fp64 inputs and strided (non-contiguous) boxes"""
    from torchvision.models.detection import _utils as det_utils

    from vision_b200 import detection as det

    def boxes(n, dt=torch.float32):
        xy = torch.rand(n, 2, device=dev) * 500
        return torch.cat([xy, xy + torch.rand(n, 2, device=dev) * 100], 1).to(dt)

    gts = [boxes(300), torch.zeros(0, 4, device=dev), boxes(3)]
    preds = [boxes(1500), boxes(77), boxes(2049).t().contiguous().t()]
    labels = [torch.randint(1, 9, (g.shape[0],), device=dev) for g in gts]
    for mode, matcher in ((det.MATCH_RAW, det_utils.Matcher(0.5, 0.4, True)), (det.MATCH_RPN, det_utils.Matcher(0.7, 0.3, True)),
                          (det.MATCH_ROI_HEADS, det_utils.Matcher(0.5, 0.5, False))):
        det.match_boxes_op(gts, preds, labels if mode == det.MATCH_ROI_HEADS else None, matcher, mode)
    det.match_boxes_op([g.half() for g in gts], [p.half() for p in preds], None, det_utils.Matcher(0.7, 0.3, True), det.MATCH_RPN)
    det.match_boxes_op([g.double() for g in gts], [p.double() for p in preds], None, det_utils.Matcher(0.7, 0.3, True), det.MATCH_RPN)


def fcos():
    """the FCOS matching kernel, memcheck only: a background image, an image without anchors, a gt count past one
    shared-memory chunk, partial last tiles, fp16 / bf16 / fp64 inputs and strided (non-contiguous) boxes"""
    from vision_b200 import detection as det

    def boxes(n, dt=torch.float32):
        xy = torch.rand(n, 2, device=dev) * 500
        return torch.cat([xy, xy + torch.rand(n, 2, device=dev) * 100], 1).to(dt)

    gts = [boxes(300), torch.zeros(0, 4, device=dev), boxes(3), boxes(5)]
    anchors = [boxes(1500), boxes(77), boxes(2049).t().contiguous().t(), boxes(0)]
    levels = [1000, 400, 100]
    det.fcos_match_op(gts, anchors, 1.5, levels)
    det.fcos_match_op([g.half() for g in gts], [a.bfloat16() for a in anchors], 1.5, levels)
    det.fcos_match_op([g.double() for g in gts], [a.double() for a in anchors], 2.5, [10**6, 0])


def retinanet_loss():
    """the head-loss kernels forward and backward, memcheck only: logits not 16-byte aligned, a row count not a multiple of
    the tile, a background image, an image with every anchor ignored, negative labels, out-of-range labels and match
    indices (which must read nothing outside labels, gt or the logits), strided anchors and gt boxes, and more images than
    one launch's descriptors"""
    from vision_b200 import detection as det

    def boxes(n):
        xy = torch.rand(n, 2, device=dev) * 500
        return torch.cat([xy, xy + torch.rand(n, 2, device=dev) * 100 + 1], 1)

    for B, A, C in ((3, 777, 91), (70, 33, 2)):
        ms = [4 if i % 3 != 1 else 0 for i in range(B)]
        gts = [boxes(m).t().contiguous().t() for m in ms]
        labels = [torch.randint(-C, C, (m,), device=dev) for m in ms]
        matched = [torch.randint(-2, max(m, 1), (A,), device=dev) for m in ms]
        matched[-1] = torch.full((A,), -2, dtype=torch.int64, device=dev)
        if ms[0]:
            labels[0][0] = C + 5
            matched[0][5] = ms[0] + 100
        logits = torch.randn(B * A * C + 1, device=dev)[1:].view(B, A, C).requires_grad_(True)
        regression = torch.randn(B, A, 4, device=dev, requires_grad=True)
        anchors = [boxes(A).t().contiguous().t() for _ in range(B)]
        (det.retinanet_cls_loss_op(logits, matched, labels) + det.retinanet_box_loss_op(regression, anchors, gts, matched,
                                                                                         [1.0, 1.0, 1.0, 1.0])).backward()


for name, fn in (("roi", roi), ("bwd", bwd), ("nms", nms), ("resize", resize), ("dcn", dcn), ("gather", gather), ("matching", matching),
                 ("fcos", fcos), ("retinanet_loss", retinanet_loss)):
    if only in ("all", name):
        fn()
        torch.cuda.synchronize()
        print(name, "done", flush=True)
