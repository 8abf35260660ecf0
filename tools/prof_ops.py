"""Small driver for ncu captures: runs one op of the hot path a few times at its BASELINE shape.
    python tools/prof_ops.py roi_align|roi_pool|ps_roi_align|ps_roi_pool|batched_nms|nms|resize|resize128|resize_noaa|deform|deform_f32|
                             roi_align_bwd|roi_align_bwd_det|roi_align_bwd14|roi_align_bwd14_det|multiscale|postprocess|preprocess [iters]
    python tools/prof_ops.py retinanet_post|fcos_post|ssd_post [iters]     fused vs. reference postprocess_detections,
                             batch 1 and 8, logits N(-4.595, 1) and N(-4.595, 0.5); select-kernel time from torch.profiler"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import vision_b200 as vb  # noqa: E402
from vision_b200 import workloads  # noqa: E402

vb._lib.load_ops()

op = sys.argv[1]
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 3
dev = "cuda"


def single_stage_post(kind: str, iters: int) -> None:
    """RetinaNet / FCOS at 800x1088 with 91 classes, SSD300: the fused method against the uninstalled one."""
    import math
    import subprocess

    from torch.profiler import ProfilerActivity, profile
    from torchvision.models.detection import _utils as det_utils
    from torchvision.models.detection.fcos import FCOS
    from torchvision.models.detection.retinanet import RetinaNet
    from torchvision.models.detection.ssd import SSD

    def bare(cls, coder, **a):
        m = cls.__new__(cls)
        m.box_coder = coder
        for k, v in a.items():
            setattr(m, k, v)
        return m

    if kind == "retinanet_post":
        model = bare(RetinaNet, det_utils.BoxCoder(weights=(1.0, 1.0, 1.0, 1.0)), score_thresh=0.05, topk_candidates=1000, nms_thresh=0.5,
                     detections_per_img=300)
    elif kind == "fcos_post":
        model = bare(FCOS, det_utils.BoxLinearCoder(normalize_by_size=True), score_thresh=0.2, topk_candidates=1000, nms_thresh=0.6,
                     detections_per_img=100)
    else:
        model = bare(SSD, det_utils.BoxCoder(weights=(10.0, 10.0, 5.0, 5.0)), score_thresh=0.01, topk_candidates=400, nms_thresh=0.45,
                     detections_per_img=200)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    print(f"{kind}: {gpu.strip().splitlines()[0] if gpu.strip() else 'unknown GPU'}")
    prior = -math.log((1 - 0.01) / 0.01)
    for batch in (1, 8):
        for sd in (1.0, 0.5):
            gen = torch.Generator(device=dev).manual_seed(0)
            if kind == "ssd_post":
                A, C, shapes = 8732, 91, [(300, 300)] * batch
                levels = [A]
                head = {"cls_logits": torch.randn(batch, A, C, generator=gen, device=dev) * sd + prior,
                        "bbox_regression": torch.randn(batch, A, 4, generator=gen, device=dev) * 0.5}
                anchors = [torch.rand(A, 4, generator=gen, device=dev).cumsum(1) * 100 for _ in shapes]
                logit_bytes = batch * A * C * 4
            else:
                a_loc = 9 if kind == "retinanet_post" else 1
                levels = [math.ceil(800 / s) * math.ceil(1088 / s) * a_loc for s in (8, 16, 32, 64, 128)]
                total, C, shapes = sum(levels), 91, [(800, 1088)] * batch
                cls = torch.randn(batch, total, C, generator=gen, device=dev) * sd + prior
                reg = torch.randn(batch, total, 4, generator=gen, device=dev) * 0.5
                head = {"cls_logits": list(cls.split(levels, 1)), "bbox_regression": list(reg.split(levels, 1))}
                if kind == "fcos_post":
                    head["bbox_ctrness"] = list(torch.randn(batch, total, 1, generator=gen, device=dev).split(levels, 1))
                anchors = [list((torch.rand(total, 4, generator=gen, device=dev).cumsum(1) * 200).split(levels)) for _ in shapes]
                logit_bytes = batch * total * C * 4
            fn = lambda: type(model).postprocess_detections(model, head, anchors, shapes)

            def timed(n):
                for _ in range(2):
                    fn()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(n):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                return e0.elapsed_time(e1) / n

            vb.uninstall()
            ref_out = fn()
            t_ref = timed(max(1, iters // 4))
            vb.install()
            try:
                got = fn()
                t_ours = timed(iters)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(iters):
                        fn()
                    torch.cuda.synchronize()
            finally:
                vb.uninstall()
            sel_us = {}
            for e in prof.key_averages():
                for name in ("ss_hist_kernel", "ss_collect_kernel", "ss_final_kernel", "ss_decode_kernel"):
                    if name in e.key:
                        sel_us[name] = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / iters
            passes = sel_us.get("ss_hist_kernel", 0.0) + sel_us.get("ss_collect_kernel", 0.0)
            bound_us = logit_bytes / 3.35e12 * 1e6
            same = all(torch.equal(a[k], b[k]) for a, b in zip(ref_out, got) for k in a)
            kernels = ", ".join(f"{k} {v:.1f} us" for k, v in sel_us.items())
            print(f"  batch {batch} N({prior:.3f}, {sd}): reference {t_ref:.3f} ms, fused {t_ours:.3f} ms ({t_ref / t_ours:.1f}x); "
                  f"{kernels}; two logit passes {passes:.1f} us vs one-read HBM bound {bound_us:.1f} us "
                  f"({bound_us / passes if passes else 0:.0%}); outputs identical: {same}")


if op in ("retinanet_post", "fcos_post", "ssd_post"):
    single_stage_post(op, iters)
    raise SystemExit(0)
if op == "roi_align":
    x, r, kw = workloads.cfg2_roi_align()
    x, r = x.to(dev), r.to(dev)
    fn = lambda: vb.ops.roi_align(x, r, **kw)
elif op == "roi_pool":
    x, r, kw = workloads.cfg2_roi_align()
    x, r = x.to(dev), r.to(dev)
    fn = lambda: vb.ops.roi_pool(x, r, 7, 0.25)
elif op in ("ps_roi_align", "ps_roi_pool"):
    x, r, kw = workloads.cfg2_roi_align()
    x, r = x[:, :245].contiguous().to(dev), r.to(dev)
    fn = (lambda: vb.ops.ps_roi_align(x, r, 7, 0.25, 2)) if op == "ps_roi_align" else (lambda: vb.ops.ps_roi_pool(x, r, 7, 0.25))
elif op in ("roi_align_bwd", "roi_align_bwd_det", "roi_align_bwd14", "roi_align_bwd14_det"):
    _, r, kw = workloads.cfg2_roi_align()
    r = r.to(dev)
    p = 14 if "bwd14" in op else 7          # 14x14: the Mask R-CNN mask head's pooled size
    g = torch.randn(1000, 256, p, p, device=dev)
    torch.use_deterministic_algorithms(op.endswith("det"))
    fn = lambda: torch.ops.vision_b200._roi_align_backward(g, r, 0.25, p, p, 1, 256, 200, 272, 2, False)
elif op == "multiscale":
    from collections import OrderedDict
    gen = torch.Generator().manual_seed(0)
    ih, iw = 800, 1088
    feats = [torch.randn(1, 256, ih // s_, iw // s_, generator=gen).to(dev) for s_ in (4, 8, 16, 32)]
    size = torch.exp(torch.rand(1000, 2, generator=gen) * 4.0 + 2.5)
    xy = torch.rand(1000, 2, generator=gen) * torch.tensor([iw, ih]) * 0.8
    rois = torch.cat([torch.zeros(1000, 1), xy, torch.minimum(xy + size, torch.tensor([float(iw), float(ih)]))], dim=1).to(dev)
    fn = lambda: torch.ops.vision_b200.multiscale_roi_align(feats, rois, [0.25, 0.125, 0.0625, 0.03125], 7, 7, 2, 2, 5, 224.0, 4.0, 1e-6)
elif op == "postprocess":
    from vision_b200 import detection
    gen = torch.Generator().manual_seed(0)
    n = 90_000
    xy = torch.rand(n, 2, generator=gen) * torch.tensor([1000.0, 760.0]); wh = torch.rand(n, 2, generator=gen) * 300 + 1
    bx = torch.cat([xy, xy + wh], 1).to(dev); sc = (torch.rand(n, generator=gen) ** 8).to(dev); lb = (torch.arange(n) % 90).to(dev)
    fn = lambda: detection.detection_postprocess(bx, sc, lb, (800, 1088), 0.05, False, 1e-2, 0.5, 100)
elif op == "preprocess":
    img = torch.randint(0, 256, (64, 3, 500, 375), dtype=torch.uint8, device=dev)
    fn = lambda: vb.transforms.classification_preprocess(img, 224, [256], (0.485, 0.456, 0.406), (0.229, 0.224, 0.225))
elif op == "batched_nms":
    b, s, i = [t.to(dev) for t in workloads.cfg3_batched_nms(clustered=len(sys.argv) > 3)]
    fn = lambda: vb.ops.batched_nms(b, s, i, 0.5)
elif op == "nms":
    b, s, i = [t.to(dev) for t in workloads.cfg3_batched_nms(n=int(os.environ.get('NMS_N', '20000')))]
    fn = lambda: vb.ops.nms(b, s, 0.5)
elif op in ("resize", "resize128", "resize_noaa", "resize_u8", "resize_f32"):
    x = workloads.cfg5_resize(device=dev, batch=128 if op == "resize128" else 32)
    if op == "resize_u8":
        x = (x.float() * 255).round().to(torch.uint8)
    if op == "resize_f32":
        x = x[:16].float()
    fn = lambda: vb.transforms.resize(x, [224, 224], antialias=(op != "resize_noaa"))
elif op in ("deform", "deform_f32"):
    dt = torch.bfloat16 if op == "deform" else torch.float32
    xi, off, w, bi, m = [t.to(dev) for t in workloads.cfg4_deform_conv2d(batch=int(os.environ.get('DCN_BATCH', '32')), dtype=dt)]
    fn = lambda: vb.ops.deform_conv2d(xi, off, w, bi, 1, 1, 1, m)
else:
    raise SystemExit(f"unknown op {op}")
for _ in range(2):
    fn()
torch.cuda.synchronize()
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
ev0.record()
for _ in range(iters):
    fn()
ev1.record()
torch.cuda.synchronize()
print(f"{op}: {ev0.elapsed_time(ev1) / iters:.4f} ms/iter over {iters} iters (warm L2)")
