"""A/B of the tensor-core deform_conv2d corner blend: fp32 FMA (default) vs the packed 16-bit HFMA2 blend (VB200_DCN_BLEND=16).
Prints, per dtype and blend, the device time of BASELINE configs[3] and the worst |err| / (1e-2 + 1e-2 |ref|) against
torchvision's CUDA fp32 kernel on the same 16-bit-rounded values.   python tools/dcn_blend_ab.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchvision as tv  # noqa: E402

import vision_b200 as vb  # noqa: E402
from vision_b200 import workloads  # noqa: E402

dev = torch.device("cuda:0")
torch.backends.cuda.matmul.allow_tf32 = False
for dt in (torch.bfloat16, torch.float16):
    for use_mask in (False, True):
        x, off, w, b, m = workloads.cfg4_deform_conv2d(device=dev, offset_scale=2.0, use_mask=use_mask)
        x, off, w, b = [t.to(dt) for t in (x, off, w, b)]
        m = None if m is None else m.to(dt)
        want = tv.ops.deform_conv2d(x.float(), off.float(), w.float(), b.float(), 1, 1, 1, None if m is None else m.float())
        bound = 1e-2 + 1e-2 * want.abs()
        for blend in ("32", "16"):
            os.environ["VB200_DCN_BLEND"] = blend
            vb._lib.core().vb200_reload_env()
            got = vb.ops.deform_conv2d(x, off, w, b, 1, 1, 1, m)
            err = (got.float() - want).abs()
            for _ in range(5):
                vb.ops.deform_conv2d(x, off, w, b, 1, 1, 1, m)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(20):
                vb.ops.deform_conv2d(x, off, w, b, 1, 1, 1, m)
            e1.record()
            torch.cuda.synchronize()
            print(f"{dt} mask={use_mask} blend={blend}: {e0.elapsed_time(e1) / 20:.3f} ms/call  worst err/bound {float((err / bound).max()):.3f} "
                  f"rms {float(err.pow(2).mean().sqrt()):.3e} max {float(err.max()):.3e}", flush=True)
