"""Generates tests/golden/*.npz from the REFERENCE implementation itself: the torchvision CPU
kernels (torch.ops.torchvision.*, CPU dispatch key) and ATen's CPU interpolate, imported in the
build container (torchvision 0.26.0+cu128 / torch 2.11.0 wheel = release build of the kernels
under /root/reference/torchvision/csrc/ops/cpu).  The fixtures pin oracle/ and the CUDA kernels.

    python tests/golden/gen_golden.py        # rewrites reference_cpu.npz and reference_cpu_resize.npz next to this script
"""
import os

import numpy as np
import torch
import torch.nn.functional as F
import torchvision
from torchvision import ops

HERE = os.path.dirname(os.path.abspath(__file__))


def make_rois(g, k, n_img, H, W, scale):
    r = torch.zeros(k, 5)
    r[:, 0] = torch.randint(0, n_img, (k,), generator=g).float()
    x1 = torch.rand(k, generator=g) * W / scale
    y1 = torch.rand(k, generator=g) * H / scale
    w = torch.rand(k, generator=g) * W / scale * 0.6 + 1
    h = torch.rand(k, generator=g) * H / scale * 0.6 + 1
    r[:, 1], r[:, 2] = x1, y1
    r[:, 3] = (x1 + w).clamp(max=W / scale + 3)
    r[:, 4] = (y1 + h).clamp(max=H / scale + 3)
    r[0, 1:] = torch.tensor([-9.0, -9.0, -5.0, -5.0])          # fully outside (empty samples)
    r[1, 1:] = torch.tensor([3.0, 3.0, 3.0, 3.0])              # degenerate
    return r


def tensors_with_iou(g, n, thr):
    # test/test_ops.py:899-914 (_create_tensors_with_iou): one engineered pair just over the threshold
    boxes = torch.rand(n, 4, generator=g) * 100
    boxes[:, 2:] += boxes[:, :2]
    boxes[-1, :] = boxes[0, :]
    x0, y0, x1, y1 = boxes[-1].tolist()
    iou_thresh = thr + 1e-5
    boxes[-1, 2] += (x1 - x0) * (1 - iou_thresh) / iou_thresh
    scores = torch.rand(n, generator=g)
    return boxes, scores


def main():
    out = {}
    g = torch.Generator().manual_seed(1234)
    # ---- nms (csrc/ops/cpu/nms_kernel.cpp) ----
    for i, thr in enumerate((0.2, 0.5, 0.8)):
        b, s = tensors_with_iou(g, 1000, thr)
        out[f"nms{i}_boxes"], out[f"nms{i}_scores"] = b.numpy(), s.numpy()
        out[f"nms{i}_thr"] = np.float64(thr)
        out[f"nms{i}_keep"] = ops.nms(b, s, thr).numpy()
    # BASELINE cfg1: 1000 random CPU boxes, thr 0.5
    torch.manual_seed(0)
    b = torch.rand(1000, 4) * 100
    b[:, 2:] += b[:, :2]
    s = torch.rand(1000)
    out["cfg1_boxes"], out["cfg1_scores"], out["cfg1_keep"] = b.numpy(), s.numpy(), ops.nms(b, s, 0.5).numpy()
    # ---- batched_nms (ops/boxes.py) ----
    for name, n, ncls in (("bnms_trick", 600, 5), ("bnms_vanilla", 3000, 7)):
        b = torch.rand(n, 4, generator=g) * 100
        b[:, 2:] = b[:, :2] + torch.rand(n, 2, generator=g) * 40 + 1
        s = torch.randperm(n, generator=g).float() / n
        idx = torch.randint(0, ncls, (n,), generator=g)
        out[f"{name}_boxes"], out[f"{name}_scores"], out[f"{name}_idxs"] = b.numpy(), s.numpy(), idx.numpy()
        out[f"{name}_keep"] = ops.batched_nms(b, s, idx, 0.5).numpy()
        out[f"{name}_keep_v"] = ops.boxes._batched_nms_vanilla(b, s, idx, 0.5).numpy()
        out[f"{name}_keep_t"] = ops.boxes._batched_nms_coordinate_trick(b, s, idx, 0.5).numpy()
    # ---- roi ops ----
    x = torch.randn(2, 10, 20, 27, generator=g)
    rois = make_rois(g, 24, 2, 20, 27, 0.25)
    out["roi_x"], out["roi_rois"] = x.numpy(), rois.numpy()
    for al in (0, 1):
        for sr in (2, -1):
            out[f"roi_align_a{al}_s{sr}"] = ops.roi_align(x, rois, (7, 5), 0.25, sr, bool(al)).numpy()
    po, pa = torch.ops.torchvision.roi_pool(x, rois, 0.25, 7, 5)
    out["roi_pool_out"], out["roi_pool_argmax"] = po.numpy(), pa.numpy()
    xp = torch.randn(2, 70, 20, 27, generator=g)
    out["psroi_x"] = xp.numpy()
    for sr in (2, -1):
        o, m = torch.ops.torchvision.ps_roi_align(xp, rois, 0.25, 7, 5, sr)
        out[f"psroi_s{sr}_out"], out[f"psroi_s{sr}_map"] = o.numpy(), m.numpy()
    # ---- deform_conv2d: the reference test's geometry (test/test_ops.py:1113-1167) ----
    B, Cin, Cout, groups, ogrps = 3, 6, 2, 2, 3
    sh, sw, ph, pw, dh, dw, kh, kw, ih, iw = 2, 1, 1, 0, 2, 1, 3, 2, 5, 4
    oh = (ih + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1
    ow = (iw + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
    inp = torch.rand(B, Cin, ih, iw, generator=g)
    off = torch.randn(B, ogrps * 2 * kh * kw, oh, ow, generator=g)
    msk = torch.randn(B, ogrps * kh * kw, oh, ow, generator=g)
    wt = torch.randn(Cout, Cin // groups, kh, kw, generator=g)
    bias = torch.randn(Cout, generator=g)
    out["dcn_x"], out["dcn_off"], out["dcn_mask"], out["dcn_w"], out["dcn_b"] = (
        inp.numpy(), off.numpy(), msk.numpy(), wt.numpy(), bias.numpy())
    out["dcn_args"] = np.array([sh, sw, ph, pw, dh, dw], dtype=np.int64)
    out["dcn_out_mask"] = ops.deform_conv2d(inp, off, wt, bias, (sh, sw), (ph, pw), (dh, dw), msk).numpy()
    out["dcn_out_nomask"] = ops.deform_conv2d(inp, off, wt, bias, (sh, sw), (ph, pw), (dh, dw), None).numpy()
    # ---- resize (ATen CPU, through F.interpolate as _geometry.py:344-350 does) ----
    img = torch.rand(2, 3, 37, 51, generator=g)
    out["rs_img"] = img.numpy()
    for mode in ("bilinear", "bicubic"):
        for aa in (0, 1):
            for size in ((12, 13), (60, 80), (37, 20)):
                out[f"rs_{mode}_aa{aa}_{size[0]}x{size[1]}"] = F.interpolate(
                    img, size=list(size), mode=mode, align_corners=False, antialias=bool(aa)).numpy()
    out["versions"] = np.array([torch.__version__, torchvision.__version__])
    # the resize arrays go to a file of their own, so that no fixture file exceeds 1 MB (tests/conftest.py merges the two)
    for name, keep in (("reference_cpu.npz", lambda k: not k.startswith("rs_")), ("reference_cpu_resize.npz", lambda k: k.startswith("rs_"))):
        part = {k: v for k, v in out.items() if keep(k)}
        np.savez_compressed(os.path.join(HERE, name), **part)
        print("wrote", os.path.join(HERE, name), len(part), "arrays")


if __name__ == "__main__":
    main()
