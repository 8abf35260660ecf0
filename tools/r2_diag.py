"""Round-2 diagnostics (GPU): (1) headroom of the 16-bit deform_conv2d tests at 1e-2, (2) timings of the reference's own
CUDA kernels (the wheel) next to ours on the five BASELINE configs.  Prints plain lines; not a test."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torchvision as tv  # noqa: E402
import vision_b200 as vb  # noqa: E402
from vision_b200 import workloads  # noqa: E402

DEV = "cuda"
flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)


def timed(fn, iters=10, warm=3, l2=True):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(iters):
        if l2:
            flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record()
        torch.cuda.synchronize()
        tot += s.elapsed_time(e)
    return tot / iters


def ratio(got, want, tol):
    err = (got.float() - want.float()).abs()
    return float((err / (tol + tol * want.float().abs())).max()), float(err.max())


def dcn_headroom():
    import oracle
    torch.manual_seed(0)
    cin, cout, g, og, sh, sw, ph, pw, dh, dw, kh, kw, ih, iw = 6, 2, 2, 3, 2, 1, 1, 0, 2, 1, 3, 2, 5, 4
    oh = (ih + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1
    ow = (iw + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
    for dtype in (torch.float16, torch.bfloat16):
        x = torch.rand(33, cin, ih, iw).to(dtype); off = torch.randn(33, og * 2 * kh * kw, oh, ow).to(dtype)
        msk = torch.randn(33, og * kh * kw, oh, ow).to(dtype); w = torch.randn(cout, cin // g, kh, kw).to(dtype); bias = torch.randn(cout).to(dtype)
        got = vb.ops.deform_conv2d(x.to(DEV), off.to(DEV), w.to(DEV), bias.to(DEV), (sh, sw), (ph, pw), (dh, dw), msk.to(DEV))
        want = torch.from_numpy(oracle.deform_conv2d(x.float().numpy(), off.float().numpy(), w.float().numpy(), bias.float().numpy(),
                                                    (sh, sw), (ph, pw), (dh, dw), msk.float().numpy()))
        print("dcn test-geometry", dtype, "ratio@1e-2, maxabs:", ratio(got.cpu(), want, 1e-2), flush=True)
    for dtype, tol in ((torch.float32, 1e-5), (torch.bfloat16, 1e-2)):
        x, off, w, b, _ = workloads.cfg4_deform_conv2d(batch=4, c_in=256, c_out=256, hw=64, dtype=dtype, offset_scale=0.0, use_mask=False)
        x, off, w, b = x.to(DEV), off.to(DEV), w.to(DEV), b.to(DEV)
        got = vb.ops.deform_conv2d(x, off, w, b, 1, 1, 1, None)
        want = torch.nn.functional.conv2d(x.double(), w.double(), b.double(), stride=1, padding=1)
        print("dcn zero-offset vs fp64 conv", dtype, f"ratio@{tol}:", ratio(got, want, tol), flush=True)


def gpu_reference():
    assert not vb.installed()
    # cfg2 roi_align
    x, rois, kw = workloads.cfg2_roi_align()
    xd, rd = x.to(DEV), rois.to(DEV)
    print("cfg2 roi_align ms: ref", timed(lambda: tv.ops.roi_align(xd, rd, **kw), 20), "ours", timed(lambda: vb.ops.roi_align(xd, rd, **kw), 20), flush=True)
    print("cfg2 roi_pool ms: ref", timed(lambda: tv.ops.roi_pool(xd, rd, 7, 0.25), 20), "ours", timed(lambda: vb.ops.roi_pool(xd, rd, 7, 0.25), 20), flush=True)
    xp = x[:, :245].contiguous().to(DEV)
    print("ps_roi_align(245ch,7x7,sr2) ms: ref", timed(lambda: tv.ops.ps_roi_align(xp, rd, 7, 0.25, 2), 20), "ours", timed(lambda: vb.ops.ps_roi_align(xp, rd, 7, 0.25, 2), 20), flush=True)
    # backward of roi_align through the reference
    xg = xd.clone().requires_grad_(True)
    o = tv.ops.roi_align(xg, rd, **kw); go = torch.randn_like(o)
    print("cfg2 roi_align backward (reference atomics) ms:", timed(lambda: torch.autograd.grad(o, xg, go, retain_graph=True), 10), flush=True)
    del xg, o, go
    go = torch.randn(1000, 256, 7, 7, device=DEV)
    t_ref = timed(lambda: torch.ops.torchvision._roi_align_backward(go, rd, 0.25, 7, 7, 1, 256, 200, 272, 2, False), 10)
    t_our = timed(lambda: torch.ops.vision_b200._roi_align_backward(go, rd, 0.25, 7, 7, 1, 256, 200, 272, 2, False), 10)
    torch.use_deterministic_algorithms(True)
    t_det = timed(lambda: torch.ops.vision_b200._roi_align_backward(go, rd, 0.25, 7, 7, 1, 256, 200, 272, 2, False), 10)
    torch.use_deterministic_algorithms(False)
    print("cfg2 _roi_align_backward op ms: ref", t_ref, "ours default (plane + smem atomics)", t_our, "ours deterministic (row-owning warps)", t_det, flush=True)
    o, am = torch.ops.torchvision.roi_pool(xd, rd, 0.25, 7, 7)
    t_ref = timed(lambda: torch.ops.torchvision._roi_pool_backward(go, rd, am, 0.25, 7, 7, 1, 256, 200, 272), 10)
    t_our = timed(lambda: torch.ops.vision_b200._roi_pool_backward(go, rd, am, 0.25, 7, 7, 1, 256, 200, 272), 10)
    print("cfg2 _roi_pool_backward op ms: ref", t_ref, "ours", t_our, flush=True)
    o, mp = torch.ops.torchvision.ps_roi_align(xp, rd, 0.25, 7, 7, 2)
    gp = torch.randn_like(o)
    t_ref = timed(lambda: torch.ops.torchvision._ps_roi_align_backward(gp, rd, mp, 0.25, 7, 7, 2, 1, 245, 200, 272), 10)
    t_our = timed(lambda: torch.ops.vision_b200._ps_roi_align_backward(gp, rd, mp, 0.25, 7, 7, 2, 1, 245, 200, 272), 10)
    print("_ps_roi_align_backward(245ch) op ms: ref", t_ref, "ours", t_our, flush=True)
    del go, o, am, mp, gp
    # cfg3
    b, s, i = [t.to(DEV) for t in workloads.cfg3_batched_nms()]
    print("cfg3 batched_nms ms: ref", timed(lambda: tv.ops.batched_nms(b, s, i, 0.5), 5, 2), "ours", timed(lambda: vb.ops.batched_nms(b, s, i, 0.5), 20), flush=True)
    for n in (1000, 20000, 100000):
        print(f"nms n={n} ms: ref", timed(lambda: tv.ops.nms(b[:n], s[:n], 0.5), 5, 2), "ours", timed(lambda: vb.ops.nms(b[:n], s[:n], 0.5), 10), flush=True)
    del b, s, i
    # cfg4
    xi, off, w, bi, m = workloads.cfg4_deform_conv2d(device=DEV)
    t_ours = timed(lambda: vb.ops.deform_conv2d(xi, off, w, bi, 1, 1, 1, m), 10)
    t16 = timed(lambda: tv.ops.deform_conv2d(xi.half(), off.half(), w.half(), bi.half(), 1, 1, 1, m.half()), 3, 1)
    xf, of, wf, bf, mf = xi.float(), off.float(), w.float(), bi.float(), m.float()
    t32 = timed(lambda: tv.ops.deform_conv2d(xf, of, wf, bf, 1, 1, 1, mf), 3, 1)
    t_ours32 = timed(lambda: vb.ops.deform_conv2d(xf, of, wf, bf, 1, 1, 1, mf), 2, 1)
    print("cfg4 deform_conv2d ms: ref fp16 (incl. casts)", t16, "ref fp32", t32, "ours bf16", t_ours, "ours fp32", t_ours32, flush=True)
    del xi, off, w, bi, m, xf, of, wf, bf, mf
    torch.cuda.empty_cache()
    # cfg5
    from torchvision.transforms.v2 import functional as TF
    img = workloads.cfg5_resize(device=DEV, batch=32)
    print("cfg5 resize batch 32 ms: ref", timed(lambda: TF.resize(img, [224, 224]), 3, 1), "ours", timed(lambda: vb.transforms.resize(img, [224, 224]), 10), flush=True)
    print("cfg5 resize bicubic batch 32 ms: ref", timed(lambda: TF.resize(img, [224, 224], interpolation=TF.InterpolationMode.BICUBIC), 3, 1),
          "ours", timed(lambda: vb.transforms.resize(img, [224, 224], interpolation=TF.InterpolationMode.BICUBIC), 5), flush=True)
    print("cfg5 resize no-AA batch 32 ms: ref", timed(lambda: TF.resize(img, [224, 224], antialias=False), 3, 1),
          "ours", timed(lambda: vb.transforms.resize(img, [224, 224], antialias=False), 5), flush=True)


def postprocess():
    import sys as _s
    _s.path.insert(0, os.path.join(ROOT, "tests"))
    from test_gpu_round2 import _reference_tail
    from vision_b200 import detection
    g = torch.Generator().manual_seed(0)
    n = 90_000                         # 1000 proposals x 90 classes, as RoIHeads.postprocess_detections sees them
    xy = torch.rand(n, 2, generator=g) * torch.tensor([1000.0, 760.0]); wh = torch.rand(n, 2, generator=g) * 300 + 1
    boxes = torch.cat([xy, xy + wh], 1).to(DEV); scores = (torch.rand(n, generator=g) ** 8).to(DEV); labels = (torch.arange(n) % 90).to(DEV)
    t_ref = timed(lambda: _reference_tail(boxes, scores, labels, (800, 1088), 0.05, False, 1e-2, 0.5, 100), 10)
    t_our = timed(lambda: detection.detection_postprocess(boxes, scores, labels, (800, 1088), 0.05, False, 1e-2, 0.5, 100), 20)
    vb.install()
    t_mid = timed(lambda: _reference_tail(boxes, scores, labels, (800, 1088), 0.05, False, 1e-2, 0.5, 100), 10)
    vb.uninstall()
    print("postprocess tail (90k candidates) ms: reference ops", t_ref, "reference ops + our batched_nms", t_mid, "fused", t_our, flush=True)


def multiscale():
    from collections import OrderedDict
    from torchvision.ops import MultiScaleRoIAlign
    g = torch.Generator().manual_seed(0)
    ih, iw = 800, 1088
    feats = OrderedDict((str(i), torch.randn(1, 256, ih // s, iw // s, generator=g).to(DEV)) for i, s in enumerate((4, 8, 16, 32)))
    size = torch.exp(torch.rand(1000, 2, generator=g) * 4.0 + 2.5)
    xy = torch.rand(1000, 2, generator=g) * torch.tensor([iw, ih]) * 0.8
    boxes = [torch.cat([xy, torch.minimum(xy + size, torch.tensor([float(iw), float(ih)]))], dim=1).to(DEV)]
    m = MultiScaleRoIAlign(["0", "1", "2", "3"], 7, 2)
    t_ref = timed(lambda: m(feats, boxes, [(ih, iw)]), 10)
    vb.install()
    t_fused = timed(lambda: m(feats, boxes, [(ih, iw)]), 20)
    from torchvision.ops import poolers
    fused = poolers._multiscale_roi_align
    poolers._multiscale_roi_align = vb._install._state["orig_msra"]
    t_loop = timed(lambda: m(feats, boxes, [(ih, iw)]), 20)
    poolers._multiscale_roi_align = fused
    vb.uninstall()
    print("MultiScaleRoIAlign 4 levels x 256 ch, 1000 boxes, ms: reference", t_ref, "ours per-level loop", t_loop, "ours fused", t_fused, flush=True)


if __name__ == "__main__":
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    if which in ("all", "dcn"):
        dcn_headroom()
    if which in ("all", "ms"):
        multiscale()
        postprocess()
    if which in ("all", "ref"):
        gpu_reference()
