"""Small driver for ncu captures: runs one op of the hot path a few times at its BASELINE shape.
    python tools/prof_ops.py roi_align|roi_pool|ps_roi_align|ps_roi_pool|batched_nms|nms|resize|resize128|resize_noaa|deform|deform_f32|
                             deform_bwd|deform_bwd_det|deform_bwd_f32|deform_bwd_det_f32|roi_align_bwd|roi_align_bwd_det|roi_align_bwd14|roi_align_bwd14_det|
                             roi_align_bwd_p2[14][_f16][_det]|multiscale|postprocess|preprocess [iters]
    python tools/prof_ops.py retinanet_post|fcos_post|ssd_post [iters]     fused vs. reference postprocess_detections,
                             batch 1 and 8, logits N(-4.595, 1) and N(-4.595, 0.5); select-kernel time from torch.profiler
    python tools/prof_ops.py keypoints_post [iters]     fused vs. reference keypointrcnn_inference, batch 1 and 8
    python tools/prof_ops.py rcnn_transform [iters]     fused vs. reference GeneralizedRCNNTransform forward + postprocess,
                             batch 1 and 8, fp32 and fp16
    python tools/prof_ops.py matching [iters]     fused vs. reference training-target assignment (RPN, RoIHeads,
                             RetinaNet), batch 2 and 8, 7 and 50 gt boxes per image
    python tools/prof_ops.py fcos [iters]     fused vs. reference FCOS.compute_loss matching, batch 2, 8 and 16, 7 and 50
                             gt boxes per image
    python tools/prof_ops.py retinanet_loss [iters]     fused vs. reference RetinaNet head losses, forward + backward,
                             batch 2 and 8, 7 and 50 gt boxes per image"""
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


def keypoints_post(iters: int) -> None:
    """Keypoint R-CNN's keypointrcnn_inference at batch 1 and 8, 100 detections per image, 17 x 56 x 56 maps N(0, 1), box
    sides U(16, 600) on 800 x 1088: the fused call against the uninstalled loop; kernel times from torch.profiler."""
    import subprocess

    from torch.profiler import ProfilerActivity, profile
    from torchvision.models.detection import roi_heads

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    print(f"keypoints_post: {gpu.strip().splitlines()[0] if gpu.strip() else 'unknown GPU'}")
    for batch in (1, 8):
        gen = torch.Generator(device=dev).manual_seed(0)
        x = torch.randn(batch * 100, 17, 56, 56, generator=gen, device=dev)
        boxes = []
        for _ in range(batch):
            wh = torch.rand(100, 2, generator=gen, device=dev) * 584 + 16
            xy = torch.rand(100, 2, generator=gen, device=dev) * (torch.tensor([1088.0, 800.0], device=dev) - wh)
            boxes.append(torch.cat([xy, xy + wh], 1))
        fn = lambda: roi_heads.keypointrcnn_inference(x, boxes)

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
        t_ref = timed(max(1, iters // 10))
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
        kern_us = {}
        for e in prof.key_averages():
            for name in ("kp_geometry_kernel", "kp_sweep_kernel", "kp_finalize_kernel"):
                if name in e.key:
                    kern_us[name] = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / iters
        # the bound from shapes: every output pixel of every resized map costs at least the 4-term y combination (4 FMAs)
        # once the row values are tabled; fp32 FMA peak of the data sheet, 67 TFLOP/s = 33.5 T FMA/s
        pixels = sum(float(((b[:, 2] - b[:, 0]).clamp(min=1).ceil() * (b[:, 3] - b[:, 1]).clamp(min=1).ceil()).sum()) for b in boxes) * 17
        bound_us = pixels * 4 / 33.5e12 * 1e6
        sweep = kern_us.get("kp_sweep_kernel", 0.0)
        same = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for ra, rb in zip(ref_out, got) for a, b in zip(ra, rb))
        kernels = ", ".join(f"{k} {v:.1f} us" for k, v in kern_us.items())
        print(f"  batch {batch}: {pixels / 1e6:.0f} M output pixels; reference {t_ref:.3f} ms, fused {t_ours:.3f} ms "
              f"({t_ref / t_ours:.0f}x); {kernels}; 4 FMA/pixel bound {bound_us:.1f} us ({bound_us / sweep if sweep else 0:.0%} of the sweep); "
              f"outputs identical: {same}")


def rcnn_transform(iters: int) -> None:
    """GeneralizedRCNNTransform (Faster R-CNN settings) forward + postprocess at batch 1 and 8 of COCO-like sizes, fp32 and fp16,
    100 boxes per image: the fused methods against the uninstalled ones.  Wall time per call ending in a synchronize, CUDA-event
    time, rcnn_batch_kernel time from torch.profiler and its share of the HBM bound (input plus padded output bytes)."""
    import subprocess
    import time

    from torch.profiler import ProfilerActivity, profile
    from torchvision.models.detection.transform import GeneralizedRCNNTransform

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    print(f"rcnn_transform: {gpu.strip().splitlines()[0] if gpu.strip() else 'unknown GPU'}")
    t = GeneralizedRCNNTransform(800, 1333, [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]).eval()
    shapes = [(480, 640), (427, 640), (640, 480), (480, 640), (500, 375), (612, 612), (480, 640), (333, 500)]
    for dtype in (torch.float32, torch.float16):
        for batch in (1, 8):
            gen = torch.Generator(device=dev).manual_seed(0)
            images = [torch.rand(3, h, w, generator=gen, device=dev).to(dtype) for h, w in shapes[:batch]]
            result = []
            for _ in range(batch):
                xy = torch.rand(100, 2, generator=gen, device=dev) * 700
                result.append({"boxes": torch.cat([xy, xy + torch.rand(100, 2, generator=gen, device=dev) * 300], 1),
                               "scores": torch.rand(100, generator=gen, device=dev),
                               "labels": torch.ones(100, dtype=torch.int64, device=dev)})
            orig = [tuple(img.shape[-2:]) for img in images]

            def fn():
                image_list, _ = t(images)
                return image_list, t.postprocess([dict(r) for r in result], image_list.image_sizes, orig)

            def timed(n):
                for _ in range(3):
                    fn()
                torch.cuda.synchronize()
                wall = []
                for _ in range(n):
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    wall.append(time.perf_counter() - t0)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(n):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                return sorted(wall)[n // 2] * 1e3, e0.elapsed_time(e1) / n

            vb.uninstall()
            ref_out = fn()
            ref_wall, ref_ev = timed(iters)
            vb.install()
            try:
                got = fn()
                wall, ev = timed(iters)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(iters):
                        fn()
                    torch.cuda.synchronize()
            finally:
                vb.uninstall()
            kern_us = {}
            for e in prof.key_averages():
                for name in ("rcnn_batch_kernel", "rcnn_rescale_kernel"):
                    if name in e.key:
                        kern_us[name] = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / iters
            nbytes = sum(img.numel() for img in images) * images[0].element_size() + got[0].tensors.numel() * got[0].tensors.element_size()
            bound_us = nbytes / 3.35e12 * 1e6
            bk = kern_us.get("rcnn_batch_kernel", 0.0)
            bits = lambda x: x.reshape(-1).view(torch.int16 if x.element_size() == 2 else torch.int32)  # noqa: E731
            same = (ref_out[0].image_sizes == got[0].image_sizes and torch.equal(bits(ref_out[0].tensors), bits(got[0].tensors))
                    and all(torch.equal(bits(a["boxes"]), bits(b["boxes"])) for a, b in zip(ref_out[1], got[1])))
            kernels = ", ".join(f"{k} {v:.1f} us" for k, v in kern_us.items())
            print(f"  {str(dtype).split('.')[-1]} batch {batch} -> {tuple(got[0].tensors.shape)}: reference wall {ref_wall:.3f} ms, "
                  f"events {ref_ev:.3f} ms; fused wall {wall:.3f} ms, events {ev:.3f} ms ({ref_wall / wall:.1f}x wall); {kernels}; "
                  f"{nbytes / 1e6:.0f} MB at 3.35 TB/s = {bound_us:.1f} us ({bound_us / bk if bk else 0:.0%} of the batch kernel); "
                  f"outputs identical: {same}")


def matching(iters: int) -> None:
    """Training-target assignment at batch 2 and 8: RegionProposalNetwork.assign_targets_to_anchors on the 217,413 RPN anchors
    of 800 x 1088 inputs with M in {7, 50} gt boxes, RoIHeads.assign_targets_to_proposals on 2000 + M proposals and the
    matching of RetinaNet.compute_loss on its 163,206 anchors; the fused methods against the uninstalled ones.  Wall time
    per call ending in a synchronize (median), and whether the outputs are identical."""
    import subprocess
    import time
    import types

    from torchvision.models.detection import _utils as det_utils, retinanet, roi_heads, rpn
    from torchvision.models.detection.anchor_utils import AnchorGenerator
    from torchvision.models.detection.image_list import ImageList
    from torchvision.ops import boxes as box_ops

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    print(f"matching: {gpu.strip().splitlines()[0] if gpu.strip() else 'unknown GPU'}")

    def anchors_for(batch, sizes, ratios, strides):
        gen = AnchorGenerator(sizes, (ratios,) * len(sizes))
        il = ImageList(torch.empty(batch, 3, 800, 1088, device=dev), [(800, 1088)] * batch)
        feats = [torch.empty(batch, 1, -(-800 // s), -(-1088 // s), device=dev) for s in strides]
        return gen(il, feats)

    head = types.SimpleNamespace(compute_loss=lambda targets, outputs, anchors, matched: matched)
    owners = {"rpn": types.SimpleNamespace(box_similarity=box_ops.box_iou, proposal_matcher=det_utils.Matcher(0.7, 0.3, True)),
              "roi_heads": types.SimpleNamespace(proposal_matcher=det_utils.Matcher(0.5, 0.5, False)),
              "retinanet": types.SimpleNamespace(proposal_matcher=det_utils.Matcher(0.5, 0.4, True), head=head)}

    def timed(fn, n):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        wall = []
        for _ in range(n):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            wall.append(time.perf_counter() - t0)
        return sorted(wall)[n // 2] * 1e3

    for batch in (2, 8):
        rpn_anchors = anchors_for(batch, ((32,), (64,), (128,), (256,), (512,)), (0.5, 1.0, 2.0), (4, 8, 16, 32, 64))
        ret_sizes = tuple((x, int(x * 2 ** (1.0 / 3)), int(x * 2 ** (2.0 / 3))) for x in (32, 64, 128, 256, 512))
        ret_anchors = anchors_for(batch, ret_sizes, (0.5, 1.0, 2.0), (8, 16, 32, 64, 128))
        for M in (7, 50):
            gen = torch.Generator(device=dev).manual_seed(M)

            def boxes(n):
                xy = torch.rand(n, 2, generator=gen, device=dev) * torch.tensor([900.0, 650.0], device=dev)
                return torch.cat([xy, xy + torch.rand(n, 2, generator=gen, device=dev) * 300 + 8], 1)

            gts = [boxes(M) for _ in range(batch)]
            labels = [torch.randint(1, 91, (M,), generator=gen, device=dev) for _ in range(batch)]
            proposals = [torch.cat([boxes(2000), g]) for g in gts]
            targets = [{"boxes": g} for g in gts]
            calls = {
                "rpn": lambda: rpn.RegionProposalNetwork.assign_targets_to_anchors(owners["rpn"], rpn_anchors, targets),
                "roi_heads": lambda: roi_heads.RoIHeads.assign_targets_to_proposals(owners["roi_heads"], proposals, gts, labels),
                "retinanet": lambda: retinanet.RetinaNet.compute_loss(owners["retinanet"], targets, {}, ret_anchors),
            }
            for name, fn in calls.items():
                vb.uninstall()
                want = fn()
                t_ref = timed(fn, iters)
                vb.install()
                try:
                    got = fn()
                    t_ours = timed(fn, iters)
                finally:
                    vb.uninstall()
                flat = lambda x: [t for part in x for t in (part if isinstance(part, (list, tuple)) else [part])]  # noqa: E731
                same = all(a.dtype == b.dtype and torch.equal(a, b) for a, b in zip(flat(want), flat(got)))
                n_pred = (rpn_anchors if name == "rpn" else ret_anchors if name == "retinanet" else proposals)[0].shape[0]
                print(f"  batch {batch}, M {M}, {name} ({n_pred} predictions per image): reference {t_ref:.3f} ms, fused {t_ours:.3f} ms "
                      f"({t_ref / t_ours:.1f}x); outputs identical: {same}")


def fcos_matching(iters: int) -> None:
    """FCOS.compute_loss at batch 2, 8 and 16 with M in {7, 50} gt boxes per image, on the 18,134 FCOS anchors of an 800 x 1088
    batch, with a head whose compute_loss returns the matched indices: the fused method against the uninstalled one.  Wall
    time per call ending in a synchronize (median), and whether the outputs are identical."""
    import subprocess
    import time
    import types

    from torchvision.models.detection import fcos
    from torchvision.models.detection.anchor_utils import AnchorGenerator
    from torchvision.models.detection.image_list import ImageList

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    print(f"fcos: {gpu.strip().splitlines()[0] if gpu.strip() else 'unknown GPU'}")
    owner = types.SimpleNamespace(center_sampling_radius=1.5,
                                  head=types.SimpleNamespace(compute_loss=lambda targets, outputs, anchors, matched: matched))
    strides = (8, 16, 32, 64, 128)

    def timed(fn, n):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        wall = []
        for _ in range(n):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            wall.append(time.perf_counter() - t0)
        return sorted(wall)[n // 2] * 1e3

    for batch in (2, 8, 16):
        gen = AnchorGenerator(tuple((s,) for s in strides), ((1.0,),) * len(strides))       # FCOS's own generator
        il = ImageList(torch.empty(batch, 3, 800, 1088, device=dev), [(800, 1088)] * batch)
        feats = [torch.empty(batch, 1, -(-800 // s), -(-1088 // s), device=dev) for s in strides]
        anchors = gen(il, feats)
        levels = [f.shape[2] * f.shape[3] for f in feats]
        for M in (7, 50):
            g = torch.Generator(device=dev).manual_seed(M)

            def boxes(n):
                xy = torch.rand(n, 2, generator=g, device=dev) * torch.tensor([900.0, 650.0], device=dev)
                return torch.cat([xy, xy + torch.rand(n, 2, generator=g, device=dev) * 300 + 8], 1)

            targets = [{"boxes": boxes(M)} for _ in range(batch)]
            fn = lambda: fcos.FCOS.compute_loss(owner, targets, {}, anchors, levels)  # noqa: E731
            vb.uninstall()
            want = fn()
            t_ref = timed(fn, iters)
            vb.install()
            try:
                got = fn()
                t_ours = timed(fn, iters)
            finally:
                vb.uninstall()
            same = all(a.dtype == b.dtype and a.stride() == b.stride() and torch.equal(a, b) for a, b in zip(want, got))
            print(f"  batch {batch}, M {M} ({anchors[0].shape[0]} anchors per image): reference {t_ref:.3f} ms, fused {t_ours:.3f} ms "
                  f"({t_ref / t_ours:.1f}x); outputs identical: {same}")


def retinanet_loss(iters: int) -> None:
    """RetinaNet's two head losses, forward + backward, on its 163,206 anchors of an 800 x 1088 batch with C = 91, batch 2 and
    8, M in {7, 50} gt boxes per image, matches from the real Matcher: the fused methods against the uninstalled ones on the
    same inputs.  Wall time per step ending in a synchronize (median), GPU kernel time per step from torch.profiler (a
    separate run), the peak-memory delta over the step and the HBM bound of the fused step computed from the shapes (the
    logits read once forward, read once and their gradient written once backward, at the data-sheet 3.35 TB/s)."""
    import re
    import subprocess
    import time

    from torch.profiler import ProfilerActivity, profile
    from torchvision.models.detection import _utils as det_utils, retinanet
    from torchvision.models.detection.anchor_utils import AnchorGenerator
    from torchvision.models.detection.image_list import ImageList
    from torchvision.ops import boxes as box_ops

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    print(f"retinanet_loss: {gpu.strip().splitlines()[0] if gpu.strip() else 'unknown GPU'}")
    C = 91
    cls_head, box_head = retinanet.RetinaNetClassificationHead(8, 9, C), retinanet.RetinaNetRegressionHead(8, 9)
    matcher = det_utils.Matcher(0.5, 0.4, True)

    def timed(fn, n):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        wall = []
        for _ in range(n):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            wall.append(time.perf_counter() - t0)
        return sorted(wall)[n // 2] * 1e3

    def kernel_ms(fn, n):
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n):
                fn()
            torch.cuda.synchronize()
        events = [e for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA]
        total = sum(e.self_device_time_total for e in events) / n / 1e3
        top = sorted(events, key=lambda e: -e.self_device_time_total)[:3]
        short = lambda k: re.sub(r"^void |vb200::|\(anonymous namespace\)::|at::native::|\(.*$", "", k)[:48]  # noqa: E731
        return total, ", ".join(f"{short(e.key)} {e.self_device_time_total / n / 1e3:.3f}" for e in top)

    def peak_mb(fn, clear):
        clear()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        return (torch.cuda.max_memory_allocated() - base) / 2**20

    sizes = tuple((x, int(x * 2 ** (1.0 / 3)), int(x * 2 ** (2.0 / 3))) for x in (32, 64, 128, 256, 512))
    for batch in (2, 8):
        gen = AnchorGenerator(sizes, ((0.5, 1.0, 2.0),) * len(sizes))
        il = ImageList(torch.empty(batch, 3, 800, 1088, device=dev), [(800, 1088)] * batch)
        anchors = gen(il, [torch.empty(batch, 1, -(-800 // s), -(-1088 // s), device=dev) for s in (8, 16, 32, 64, 128)])
        A = anchors[0].shape[0]
        for M in (7, 50):
            g = torch.Generator(device=dev).manual_seed(M)
            targets, matched = [], []
            for a in anchors:
                xy = torch.rand(M, 2, generator=g, device=dev) * torch.tensor([900.0, 650.0], device=dev)
                boxes = torch.cat([xy, xy + torch.rand(M, 2, generator=g, device=dev) * 300 + 8], 1)
                targets.append({"boxes": boxes, "labels": torch.randint(1, C, (M,), generator=g, device=dev)})
                matched.append(matcher(box_ops.box_iou(boxes, a)))
            logits = (torch.randn(batch, A, C, generator=g, device=dev) - 4.595).requires_grad_(True)
            regression = (torch.randn(batch, A, 4, generator=g, device=dev) * 0.1).requires_grad_(True)

            def clear():
                logits.grad = regression.grad = None

            def step():
                clear()
                loss = (cls_head.compute_loss(targets, {"cls_logits": logits}, matched)
                        + box_head.compute_loss(targets, {"bbox_regression": regression}, anchors, matched))
                loss.backward()
                return loss.detach()

            rows = {}
            for name in ("reference", "fused"):
                if name == "fused":
                    vb.install()
                try:
                    loss = step()
                    rows[name] = (loss, logits.grad.clone(), regression.grad.clone(), timed(step, iters), kernel_ms(step, 5),
                                  peak_mb(step, clear))
                finally:
                    vb.uninstall()
            bound_us = batch * A * C * 4 * 3 / 3.35e12 * 1e6
            (l0, gc0, gr0, *_), (l1, gc1, gr1, *_) = rows["reference"], rows["fused"]
            print(f"  batch {batch}, M {M} ({A} anchors per image, {int(sum((m >= 0).sum() for m in matched))} foreground): "
                  f"HBM bound of the fused step {bound_us:.0f} us; loss {l0.item():.6f} vs {l1.item():.6f}, "
                  f"max |d grad| cls {(gc0 - gc1).abs().max().item():.2e}, box {(gr0 - gr1).abs().max().item():.2e}")
            for name, (_, _, _, wall, (kern, top), peak) in rows.items():
                print(f"    {name:9s} wall {wall:.3f} ms per step, kernels {kern:.3f} ms ({top}), peak +{peak:.0f} MiB")


if op == "retinanet_loss":
    retinanet_loss(iters)
    raise SystemExit(0)
if op == "matching":
    matching(iters)
    raise SystemExit(0)
if op == "fcos":
    fcos_matching(iters)
    raise SystemExit(0)
if op == "rcnn_transform":
    rcnn_transform(iters)
    raise SystemExit(0)
if op in ("retinanet_post", "fcos_post", "ssd_post"):
    single_stage_post(op, iters)
    raise SystemExit(0)
if op == "keypoints_post":
    keypoints_post(iters)
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
elif op.startswith("roi_align_bwd_p2"):
    # FPN P2 of a padded 800 x 1344 batch of 2 (2 x 256 x 192 x 336; an fp32 plane does not fit in shared memory), 1000 RoIs,
    # sr 2: roi_align_bwd_p2[14][_f16][_det] - 14x14 bins (mask head) instead of 7x7, fp16 instead of fp32, deterministic mode
    gen = torch.Generator().manual_seed(0)
    p = 14 if "p214" in op else 7
    dt = torch.float16 if "_f16" in op else torch.float32
    wh = torch.exp(torch.rand(1000, 2, generator=gen) * 3.0 + 2.5)
    xy = torch.rand(1000, 2, generator=gen) * torch.tensor([1344.0, 768.0]) * 0.9
    r = torch.cat([torch.randint(0, 2, (1000, 1), generator=gen).float(), xy, xy + wh], 1).to(dt).to(dev)
    g = torch.randn(1000, 256, p, p, device=dev).to(dt)
    torch.use_deterministic_algorithms(op.endswith("_det"))
    fn = lambda: torch.ops.vision_b200._roi_align_backward(g, r, 0.25, p, p, 2, 256, 192, 336, 2, False)
    gpu = torch.cuda.get_device_name()
    try:
        import subprocess
        gpu += ", power limit " + subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                                                 text=True).stdout.strip().splitlines()[0]
    except Exception:
        pass
    print(f"{op}: {gpu}")
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
elif op in ("deform_bwd", "deform_bwd_det", "deform_bwd_f32", "deform_bwd_det_f32"):
    # the whole deform_conv2d backward (two GEMMs + our kernels) at cfg4; _det: grad_input by the deterministic gather
    import warnings
    dt = torch.float32 if op.endswith("_f32") else torch.bfloat16
    xi, off, w, bi, m = [t.to(dev) for t in workloads.cfg4_deform_conv2d(batch=int(os.environ.get('DCN_BATCH', '32')), dtype=dt)]
    g = torch.randn(xi.shape[0], w.shape[0], xi.shape[2], xi.shape[3], device=dev).to(dt)
    torch.use_deterministic_algorithms("_det" in op, warn_only=True)        # warn_only: the shim's GEMMs are cuBLAS
    warnings.simplefilter("ignore", UserWarning)
    fn = lambda: torch.ops.vision_b200._deform_conv2d_backward(g, xi, w, off, m, bi, 1, 1, 1, 1, 1, 1, 1, 1, True)
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
