"""GPU parity tests added in round 2 (run on an H100: `pytest -m gpu`).

* fp16 nms / batched_nms: bit-exact against the reference's own CUDA kernel (devIoU<Half>,
  csrc/ops/cuda/nms_kernel.cu:42-54; the in-half coordinate trick, ops/boxes.py:92-109) and the oracle's half mode;
* score-order edge cases (+-0.0 ties, NaN, +-inf, many ties) against aten::sort(stable, descending) as the reference uses it;
* deform_conv2d at BASELINE configs[3] FULL size (N=32, 512->512, 64x64, bf16) against the reference CUDA op run in
  fp32 on the bf16-rounded inputs, tolerance 1e-2 as north_star states.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def npy(x):
    return x.detach().float().cpu().numpy() if x.is_floating_point() else x.detach().cpu().numpy()


def _fp16_boxes(n, seed, span=600.0, clustered=True):
    g = torch.Generator().manual_seed(seed)
    if clustered:
        c = max(1, n // 12)
        cxy = torch.rand(c, 2, generator=g) * span
        cwh = torch.rand(c, 2, generator=g) * 120 + 4
        rep = torch.arange(n) % c
        xy = cxy[rep] + torch.randn(n, 2, generator=g) * 0.08 * cwh[rep]
        wh = cwh[rep] * (1 + torch.randn(n, 2, generator=g) * 0.08).clamp(min=0.3)
    else:
        xy = torch.rand(n, 2, generator=g) * span
        wh = torch.rand(n, 2, generator=g) * 150 + 1
    boxes = torch.cat([xy, xy + wh], dim=1).half()
    scores = torch.rand(n, generator=g).half()          # fp16 scores: thousands of exact ties -> the stable order matters
    return boxes, scores


@pytest.mark.parametrize("thr", [0.3, 0.5, 0.7])
def test_nms_float16_bit_exact_vs_reference_cuda(vb, oracle, thr):
    tv = pytest.importorskip("torchvision")
    assert not vb.installed()
    for n, clustered in ((12_000, True), (20_000, False), (777, True)):
        b, s = _fp16_boxes(n, seed=n, clustered=clustered)
        bd, sd = b.to(DEV), s.to(DEV)
        ref = tv.ops.nms(bd, sd, thr)                               # reference CUDA kernel, devIoU<Half>
        ours = vb.ops.nms(bd, sd, thr)
        assert ours.dtype == torch.int64 and torch.equal(ref, ours)
        want = oracle.nms(b.float().numpy(), s.float().numpy(), thr, mode=oracle.NMS_MODE_CUDA_HALF)
        assert np.array_equal(npy(ours), want)


def test_batched_nms_float16_bit_exact_vs_reference_cuda(vb, oracle):
    tv = pytest.importorskip("torchvision")
    assert not vb.installed()
    g = torch.Generator().manual_seed(5)
    # (a) coordinate trick in half (numel <= 100k): 80 classes x max coordinate ~720 overflows fp16 for the high class ids
    # (offsets become inf) - reproduced literally; (b) few classes: no overflow; (c) vanilla (numel > 100k): per-class devIoU<Half>
    for n, classes in ((20_000, 80), (24_000, 12), (30_000, 80)):
        b, s = _fp16_boxes(n, seed=n + classes)
        idx = torch.randint(0, classes, (n,), generator=g)
        bd, sd, idd = b.to(DEV), s.to(DEV), idx.to(DEV)
        ref = tv.ops.batched_nms(bd, sd, idd, 0.5)
        ours = vb.ops.batched_nms(bd, sd, idd, 0.5)
        if 4 * n <= 100_000:
            assert torch.equal(ref, ours)
        else:
            # vanilla: the reference's final sort is unstable (boxes.py:126), so tied fp16 scores may be permuted:
            # same set, same score sequence, and our order is the stable one
            assert torch.equal(torch.sort(ref)[0], torch.sort(ours)[0])
            assert torch.equal(sd[ref], sd[ours])
        want = oracle.batched_nms(b.float().numpy(), s.float().numpy(), idx.numpy(), 0.5, mode=oracle.NMS_MODE_CUDA_HALF,
                                  device_is_cuda=True)
        assert np.array_equal(npy(ours), want)
    # through the installed API surface (torchvision.ops.batched_nms rebinding keeps fp16 on our kernels)
    vb.install()
    try:
        before = vb.launch_count()
        again = tv.ops.batched_nms(bd, sd, idd, 0.5)
        assert vb.launch_count() > before and torch.equal(again, ours)
    finally:
        vb.uninstall()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.float16])
def test_nms_score_order_edge_cases_vs_reference_cuda(vb, dtype):
    """aten::sort(stable=True, descending=True) semantics of nms_kernel.cu:200: -0.0 == +0.0 (index order kept), NaN scores
    first, +-inf at the ends, long runs of ties.  Small (bitonic path of torch) and large (radix path) sizes."""
    tv = pytest.importorskip("torchvision")
    assert not vb.installed()
    for n in (300, 9000):
        g = torch.Generator().manual_seed(n)
        xy = torch.rand(n, 2, generator=g) * 200
        wh = torch.rand(n, 2, generator=g) * 60 + 2
        boxes = torch.cat([xy, xy + wh], dim=1).to(dtype)
        s = (torch.randint(0, 6, (n,), generator=g).float() - 2.0) * 0.25          # values in {-0.5..0.75}: heavy ties, zeros
        s[torch.rand(n, generator=g) < 0.1] = -0.0
        s[torch.rand(n, generator=g) < 0.1] = 0.0
        s[torch.rand(n, generator=g) < 0.02] = float("inf")
        s[torch.rand(n, generator=g) < 0.02] = float("-inf")
        s[torch.rand(n, generator=g) < 0.02] = float("nan")                         # positive quiet NaN
        s = s.to(dtype)
        bd, sd = boxes.to(DEV), s.to(DEV)
        ref = tv.ops.nms(bd, sd, 0.5)
        ours = vb.ops.nms(bd, sd, 0.5)
        assert torch.equal(ref, ours), (n, dtype)


@pytest.mark.parametrize("variant", ["mask", "nomask", "zero_offset"])
def test_deform_conv2d_cfg4_full_size_vs_reference_cuda(vb, oracle, variant):
    """BASELINE configs[3] at FULL size through the wgmma kernel the bench times (BN=256, 3 stages, two consumer warpgroups):
    N=32, 512->512, 64x64, 3x3, bf16.  Reference = torchvision's CUDA deform_conv2d in fp32 on the bf16-rounded values
    (the reference has no bf16 kernel on any backend), tolerance 1e-2 (north_star).  One image is also checked
    against the CPU oracle."""
    tv = pytest.importorskip("torchvision")
    from vision_b200 import workloads

    assert not vb.installed()
    x, off, w, b, m = workloads.cfg4_deform_conv2d(device=DEV, offset_scale=0.0 if variant == "zero_offset" else 2.0,
                                                   use_mask=(variant == "mask"))
    before = vb.launch_count()
    got = vb.ops.deform_conv2d(x, off, w, b, 1, 1, 1, m)
    assert vb.launch_count() > before and got.dtype == torch.bfloat16 and got.shape == (32, 512, 64, 64)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        want = tv.ops.deform_conv2d(x.float(), off.float(), w.float(), b.float(), 1, 1, 1, None if m is None else m.float())
        if variant == "zero_offset":
            oldc = torch.backends.cudnn.allow_tf32
            torch.backends.cudnn.allow_tf32 = False
            conv = torch.nn.functional.conv2d(x.float(), w.float(), b.float(), stride=1, padding=1)
            torch.backends.cudnn.allow_tf32 = oldc
            np.testing.assert_allclose(npy(want), npy(conv), rtol=1e-4, atol=1e-4)       # sanity of the reference itself
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    err = (got.float() - want).abs()
    bound = 1e-2 + 1e-2 * want.abs()
    worst = float((err / bound).max())
    assert worst <= 1.0, f"max |err| / (1e-2 + 1e-2 |ref|) = {worst:.3f}, max abs err {float(err.max()):.4g}"
    # CPU oracle on the last image (fp32 arithmetic in the reference CPU kernel's order)
    sl = slice(31, 32)
    want_cpu = oracle.deform_conv2d(npy(x[sl]), npy(off[sl]), npy(w), npy(b), (1, 1), (1, 1), (1, 1), None if m is None else npy(m[sl]))
    np.testing.assert_allclose(npy(got[sl]), want_cpu, rtol=1e-2, atol=1e-2)


# =============================== roi_pool / ps_roi_align forward: new plane-major kernels ===============================
def _rois(k, b, h, w, scale, seed, small=False):
    g = torch.Generator().manual_seed(seed)
    ih, iw = h / scale, w / scale
    x1 = torch.rand(k, generator=g) * iw * 1.1 - 0.05 * iw        # a few RoIs start outside the image
    y1 = torch.rand(k, generator=g) * ih * 1.1 - 0.05 * ih
    span = 0.08 if small else 0.6
    bw = torch.rand(k, generator=g) * iw * span + 0.2
    bh = torch.rand(k, generator=g) * ih * span + 0.2
    return torch.stack([torch.randint(0, b, (k,), generator=g).float(), x1, y1, x1 + bw, y1 + bh], dim=1)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.float16])
def test_roi_pool_plane_major_shapes_bit_exact_vs_reference_cuda(vb, oracle, dtype):
    """Every lane mapping of roi_pool_plane_kernel (Q = 32 / PW sub-lanes: PW 1, 2, 5, 7, 16, 17, 40) on resident and
    non-resident planes, batch > 1, RoIs partly outside, empty bins: output AND argmax identical to the reference."""
    tv = pytest.importorskip("torchvision")
    assert not vb.installed()
    cases = [((2, 5, 40, 52), 300, (7, 7), 0.25), ((1, 3, 30, 30), 1200, (5, 5), 0.5), ((3, 4, 25, 33), 200, (3, 17), 1.0),
             ((1, 2, 64, 48), 2000, (2, 40), 0.5), ((2, 6, 20, 20), 40, (1, 1), 1.0), ((1, 8, 200, 272), 600, (7, 7), 0.25),
             ((1, 2, 64, 480), 300, (2, 20), 1.0),                        # Q = 1 and bins wider than 8 columns: the plain-loop branch
             ((1, 2, 300, 400), 100, (4, 2), 0.25)]                      # last: fp32 plane 480 KB > shared memory
    for shape, k, (ph, pw), scale in cases:
        b, c, h, w = shape
        g = torch.Generator().manual_seed(k + pw)
        x = torch.randn(*shape, generator=g)
        x[:, :, ::3, ::4] = 0.75                                          # exact ties: the first maximum in row-major order wins
        x[:, :, 1::5, 2::7] = float("nan")                                 # NaN is never selected (v > best is false)
        x[:, 0, :4, :] = -0.0                                              # signed zeros: the first one's sign is what comes out
        rois = _rois(k, b, h, w, scale, seed=k)
        xd, rd = x.to(dtype).to(DEV), rois.to(dtype).to(DEV)
        o1, a1 = torch.ops.torchvision.roi_pool(xd, rd, scale, ph, pw)
        o2, a2 = torch.ops.vision_b200.roi_pool(xd, rd, scale, ph, pw)
        assert torch.equal(a1, a2), (shape, ph, pw, dtype)
        assert torch.equal(o1, o2), (shape, ph, pw, dtype)
    if dtype == torch.float32:
        wo, wa = oracle.roi_pool(x.numpy(), rois.numpy(), (ph, pw), scale)
        assert np.array_equal(npy(o2), wo) and np.array_equal(npy(a2), wa)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.float16])
def test_ps_roi_align_plane_major_vs_reference(vb, oracle, dtype):
    tv = pytest.importorskip("torchvision")
    assert not vb.installed()
    for shape, k, (ph, pw), scale, sr in [((2, 50, 30, 40), 500, (5, 5), 0.5, 2), ((1, 245, 40, 52), 1500, (7, 7), 0.25, 2),
                                         ((1, 18, 64, 64), 64, (3, 3), 1.0, -1), ((2, 8, 20, 24), 3000, (2, 2), 0.5, 3)]:
        b, c, h, w = shape
        g = torch.Generator().manual_seed(k)
        x = torch.randn(*shape, generator=g)
        rois = _rois(k, b, h, w, scale, seed=k + 1)
        xd, rd = x.to(dtype).to(DEV), rois.to(dtype).to(DEV)
        o1, m1 = torch.ops.torchvision.ps_roi_align(xd, rd, scale, ph, pw, sr)
        o2, m2 = torch.ops.vision_b200.ps_roi_align(xd, rd, scale, ph, pw, sr)
        assert torch.equal(m1, m2)
        # fp16: the reference rounds EVERY scalar op to half (coordinates included); we compute in fp32 from the same fp16
        # inputs, so the comparison bound is the reference's own coordinate rounding (2^-11 of a coordinate ~ 50 px)
        if dtype == torch.float16:
            # ground truth for 16-bit storage = the reference arithmetic in fp32 on the same fp16 values (as north_star
            # defines it for bf16 deform_conv2d); the reference's own Half kernel is only required to be no closer to it
            truth = torch.ops.torchvision.ps_roi_align(xd.float(), rd.float(), scale, ph, pw, sr)[0]
            err, err_ref = (o2.float() - truth).abs(), (o1.float() - truth).abs()
            bound = 1e-2 + 1e-2 * truth.abs()
            assert float((err / bound).max()) <= 1.0, (float(err.max()), float(err_ref.max()))
        else:
            tol = dict(rtol=1e-5, atol=1e-5) if dtype == torch.float64 else dict(rtol=1e-5, atol=1e-4)
            # fp32: the compiled CUDA reference contracts its coordinate arithmetic and is itself ~1e-5 from its CPU kernel (DESIGN.md §2)
            np.testing.assert_allclose(npy(o2), npy(o1), **tol)
        if dtype == torch.float32:
            want, wm = oracle.ps_roi_align(x.numpy(), rois.numpy(), (ph, pw), scale, sr)
            assert np.array_equal(npy(o2), want) and np.array_equal(npy(m2), wm)       # bit-exact vs the CPU reference arithmetic


# =============================== backward kernels (SURVEY §8f1) ===============================
def _bwd_case(seed, b, c, h, w, k, small=False, scale=0.25):
    g = torch.Generator().manual_seed(seed)
    rois = _rois(k, b, h, w, scale, seed=seed + 7, small=small)
    return g, rois


@pytest.mark.parametrize("aligned", [False, True])
@pytest.mark.parametrize("sr", [1, 2, 3])
def test_roi_align_backward_plane_path_vs_reference_and_deterministic(vb, aligned, sr):
    """fp32 plane-resident backward: close to the reference CUDA backward run in fp64 (ground truth), at least as close as
    the reference's own fp32 atomics kernel, bit-identical between two runs, and equal (to rounding) to our atomic kernel."""
    tv = pytest.importorskip("torchvision")
    assert not vb.installed()
    from test_gpu_parity import force_env
    for (b, c, h, w, k, ph, pw, small) in [(2, 6, 50, 68, 700, 7, 7, False), (1, 3, 24, 30, 400, 7, 7, True), (1, 2, 40, 40, 300, 3, 20, False),
                                           (3, 2, 9, 11, 100, 2, 2, False)]:
        g, rois = _bwd_case(b * 100 + k + sr, b, c, h, w, k, small=small)
        grad = torch.randn(k, c, ph, pw, generator=g) * 0.25
        gd, rd = grad.to(DEV), rois.to(DEV)
        args = (0.25, ph, pw, b, c, h, w, sr, aligned)
        truth = torch.ops.torchvision._roi_align_backward(gd.double(), rd.double(), *args)
        ref32 = torch.ops.torchvision._roi_align_backward(gd, rd, *args)
        before = vb.launch_count()
        fast = torch.ops.vision_b200._roi_align_backward(gd, rd, *args)          # default: resident plane + shared-memory atomics
        assert vb.launch_count() > before and fast.shape == (b, c, h, w) and fast.dtype == torch.float32
        scale_ = truth.abs().max().item() + 1e-12
        np.testing.assert_allclose(npy(fast), truth.float().cpu().numpy(), rtol=1e-5, atol=1e-5 * max(1.0, scale_))
        torch.use_deterministic_algorithms(True)          # the reference raises in this mode; ours switches to the row-owning kernel
        try:
            ours = torch.ops.vision_b200._roi_align_backward(gd, rd, *args)
            again = torch.ops.vision_b200._roi_align_backward(gd, rd, *args)
        finally:
            torch.use_deterministic_algorithms(False)
        assert torch.equal(ours, again)                                        # bit-reproducible
        err = (ours.double() - truth).abs().max().item()
        err_ref = (ref32.double() - truth).abs().max().item()
        assert err <= 1e-5 * (1 + scale_), (err, err_ref, scale_)
        np.testing.assert_allclose(npy(ours), truth.float().cpu().numpy(), rtol=1e-5, atol=1e-5 * max(1.0, scale_))
        with force_env("VB200_ROI_BWD_PATH", "atomic"):
            atom = torch.ops.vision_b200._roi_align_backward(gd, rd, *args)
        np.testing.assert_allclose(npy(atom), truth.float().cpu().numpy(), rtol=1e-5, atol=1e-5 * max(1.0, scale_))


@pytest.mark.parametrize("dtype", [torch.float64, torch.float16])
def test_roi_align_backward_other_dtypes_and_adaptive_grid(vb, dtype):
    tv = pytest.importorskip("torchvision")
    assert not vb.installed()
    b, c, h, w, k = 2, 4, 20, 26, 150
    g, rois = _bwd_case(11, b, c, h, w, k)
    grad = (torch.randn(k, c, 5, 5, generator=g) * 0.25).to(dtype).to(DEV)
    rd = rois.to(dtype).to(DEV)
    for sr in (2, -1):
        args = (0.25, 5, 5, b, c, h, w, sr, False)
        ours = torch.ops.vision_b200._roi_align_backward(grad, rd, *args)
        assert ours.dtype == dtype
        if dtype == torch.float64:
            ref = torch.ops.torchvision._roi_align_backward(grad, rd, *args)
            np.testing.assert_allclose(ours.cpu().numpy(), ref.cpu().numpy(), rtol=1e-9, atol=1e-9)
        else:
            # fp16: both kernels round every atomic add to half, and the reference also rounds its coordinates to half; the
            # ground truth is the fp64 scatter of the same fp16 values - bound: a few half ulps of the largest accumulated value
            truth = torch.ops.torchvision._roi_align_backward(grad.double(), rd.double(), *args)
            ref = torch.ops.torchvision._roi_align_backward(grad, rd, *args)
            bound = 4e-3 * max(1.0, truth.abs().max().item()) * 8
            err, err_ref = (ours.double() - truth).abs().max().item(), (ref.double() - truth).abs().max().item()
            assert err <= max(bound, 2 * err_ref), (err, err_ref, bound)
    # fp32 adaptive grid takes the atomic kernel too
    g32, r32 = grad.float(), rd.float()
    args = (0.25, 5, 5, b, c, h, w, -1, True)
    np.testing.assert_allclose(npy(torch.ops.vision_b200._roi_align_backward(g32, r32, *args)),
                               npy(torch.ops.torchvision._roi_align_backward(g32.double(), r32.double(), *args).float()), rtol=1e-5, atol=1e-5)


def test_roi_pool_and_ps_roi_align_backward_vs_reference(vb):
    tv = pytest.importorskip("torchvision")
    assert not vb.installed()
    for (b, c, h, w, k, p) in [(2, 5, 40, 52, 600, 7), (1, 3, 16, 16, 900, 2), (1, 2, 300, 400, 50, 3)]:
        g, rois = _bwd_case(k, b, c, h, w, k)
        x = torch.randn(b, c, h, w, generator=g)
        x[:, :, ::2, ::2] = 1.5                                        # ties: neighbouring bins share their argmax
        xd, rd = x.to(DEV), rois.to(DEV)
        out, am = torch.ops.torchvision.roi_pool(xd, rd, 0.25, p, p)
        grad = torch.randn(out.shape, generator=g).to(DEV) * 0.25
        args = (0.25, p, p, b, c, h, w)
        truth = torch.ops.torchvision._roi_pool_backward(grad.double(), rd.double(), am, *args)
        fast = torch.ops.vision_b200._roi_pool_backward(grad, rd, am, *args)                 # atomic scatter (default)
        np.testing.assert_allclose(npy(fast), truth.float().cpu().numpy(), rtol=1e-5, atol=1e-5 * max(1.0, truth.abs().max().item()))
        torch.use_deterministic_algorithms(True)        # the reference raises here (alertNotDeterministic); ours switches kernels
        try:
            ours = torch.ops.vision_b200._roi_pool_backward(grad, rd, am, *args)
            if h * w * 4 < 200_000:                     # plane fits shared memory -> the row-owning kernel, bit-reproducible
                assert torch.equal(ours, torch.ops.vision_b200._roi_pool_backward(grad, rd, am, *args))
        finally:
            torch.use_deterministic_algorithms(False)
        np.testing.assert_allclose(npy(ours), truth.float().cpu().numpy(), rtol=1e-5, atol=1e-5 * max(1.0, truth.abs().max().item()))
    for (b, cout, h, w, k, p, sr) in [(2, 3, 30, 40, 500, 5, 2), (1, 2, 20, 20, 800, 3, 1), (1, 1, 300, 400, 40, 2, 2)]:
        c = cout * p * p
        g, rois = _bwd_case(k + p, b, c, h, w, k)
        rd = rois.to(DEV)
        xd = torch.randn(b, c, h, w, generator=g).to(DEV)
        out, mapping = torch.ops.torchvision.ps_roi_align(xd, rd, 0.25, p, p, sr)
        grad = torch.randn(out.shape, generator=g).to(DEV) * 0.25
        args = (0.25, p, p, sr, b, c, h, w)
        truth = torch.ops.torchvision._ps_roi_align_backward(grad.double(), rd.double(), mapping, *args)
        fast = torch.ops.vision_b200._ps_roi_align_backward(grad, rd, mapping, *args)        # atomic scatter (default)
        np.testing.assert_allclose(npy(fast), truth.float().cpu().numpy(), rtol=1e-5, atol=1e-5 * max(1.0, truth.abs().max().item()))
        torch.use_deterministic_algorithms(True)
        try:
            ours = torch.ops.vision_b200._ps_roi_align_backward(grad, rd, mapping, *args)
            if h * w * 4 < 200_000:
                assert torch.equal(ours, torch.ops.vision_b200._ps_roi_align_backward(grad, rd, mapping, *args))
        finally:
            torch.use_deterministic_algorithms(False)
        np.testing.assert_allclose(npy(ours), truth.float().cpu().numpy(), rtol=1e-5, atol=1e-5 * max(1.0, truth.abs().max().item()))


def test_autograd_through_both_api_surfaces(vb):
    """(1) vision_b200.ops.* are differentiable (autograd formulas registered on the vision_b200:: ops);
    (2) after install() torchvision.ops.roi_align(...).backward() runs OUR backward kernel (launch counter) and matches the
    reference's gradient; gradcheck in fp64 mirrors test/test_ops.py:193-217."""
    tv = pytest.importorskip("torchvision")
    from torch.autograd import gradcheck
    from vision_b200 import workloads

    assert not vb.installed()
    x, rois, kw = workloads.cfg2_roi_align(channels=16, k=300)
    xd, rd = x.to(DEV), rois.to(DEV)
    xr = xd.clone().requires_grad_(True)
    tv.ops.roi_align(xr, rd, **kw).square().sum().backward()
    ref_grad = xr.grad.clone()
    xo = xd.clone().requires_grad_(True)
    vb.ops.roi_align(xo, rd, **kw).square().sum().backward()
    np.testing.assert_allclose(npy(xo.grad), npy(ref_grad), rtol=1e-4, atol=1e-4 * ref_grad.abs().max().item())
    vb.install()
    try:
        xi = xd.clone().requires_grad_(True)
        before = vb.launch_count()
        out = tv.ops.roi_align(xi, rd, **kw)
        mid = vb.launch_count()
        out.square().sum().backward()
        assert mid > before and vb.launch_count() > mid                       # forward AND backward ran on our kernels
        np.testing.assert_allclose(npy(xi.grad), npy(ref_grad), rtol=1e-4, atol=1e-4 * ref_grad.abs().max().item())
        for op, extra in ((tv.ops.roi_pool, {}), (tv.ops.ps_roi_align, dict(sampling_ratio=2))):
            xp = torch.randn(1, 18, 20, 24, device=DEV, requires_grad=True)
            r = torch.tensor([[0, 2.0, 3.0, 60.0, 50.0], [0, 10.0, 10.0, 30.0, 70.0]], device=DEV)
            before = vb.launch_count()
            op(xp, r, 3, 0.25, **extra).sum().backward()
            assert vb.launch_count() >= before + 2 and xp.grad.abs().sum().item() > 0
    finally:
        vb.uninstall()
    # gradcheck, fp64 (the reference's test shapes)
    torch.manual_seed(0)
    xg = torch.rand(1, 8, 5, 5, dtype=torch.float64, device=DEV, requires_grad=True)
    r = torch.tensor([[0, 0, 0, 4, 4], [0, 0, 2, 3, 4], [0, 2, 2, 4, 4]], dtype=torch.float64, device=DEV)
    assert gradcheck(lambda z: vb.ops.roi_align(z, r, 2, spatial_scale=1, sampling_ratio=1), (xg,), atol=1e-5)
    assert gradcheck(lambda z: vb.ops.ps_roi_align(z, r, 2, spatial_scale=1, sampling_ratio=1), (xg,), atol=1e-5)
    assert gradcheck(lambda z: vb.ops.roi_pool(z, r, 2, spatial_scale=1), (xg,), atol=1e-5)


# =============================== fused MultiScaleRoIAlign (SURVEY §8f2) ===============================
def _fpn_case(batch=2, channels=32, seed=0, n_boxes=(700, 500)):
    from collections import OrderedDict

    g = torch.Generator().manual_seed(seed)
    ih, iw = 800, 1088
    feats = OrderedDict()
    for name, s in (("0", 4), ("1", 8), ("2", 16), ("3", 32)):
        feats[name] = torch.randn(batch, channels, ih // s, iw // s, generator=g)
    boxes = []
    for n in n_boxes[:batch]:
        size = torch.exp(torch.rand(n, 2, generator=g) * 4.6 + 2.0)            # 7 .. 730 px: every level is hit
        xy = torch.rand(n, 2, generator=g) * torch.tensor([iw, ih]) * 0.9
        b = torch.cat([xy, torch.minimum(xy + size, torch.tensor([float(iw), float(ih)]))], dim=1)
        # exact LevelMapper boundaries (sqrt(area) = 112, 224, 448 -> log2 ratios -1, 0, 1), a zero-area and an inverted box
        b[0] = torch.tensor([10.0, 10.0, 122.0, 122.0]); b[1] = torch.tensor([10.0, 10.0, 234.0, 234.0])
        b[2] = torch.tensor([10.0, 10.0, 458.0, 458.0]); b[3] = torch.tensor([50.0, 60.0, 50.0, 90.0])
        b[4] = torch.tensor([300.0, 200.0, 250.0, 260.0]); b[5] = torch.tensor([0.0, 0.0, 224.0 * 2, 112.0])
        boxes.append(b)
    return feats, boxes, [(ih, iw)] * batch


def test_multiscale_roi_align_fused_vs_reference(vb):
    tv = pytest.importorskip("torchvision")
    from torchvision.ops import MultiScaleRoIAlign
    from torchvision.ops.poolers import _convert_to_roi_format

    assert not vb.installed()
    feats, boxes, shapes = _fpn_case()
    fd = type(feats)((k, v.to(DEV)) for k, v in feats.items())
    bd = [b.to(DEV) for b in boxes]
    m = MultiScaleRoIAlign(["0", "1", "2", "3"], 7, 2)
    ref_cuda = m(fd, bd, shapes)                                     # reference: per-level loop on its own CUDA kernels
    ref_levels = m.map_levels(bd)
    # the reference CPU kernel on the reference's own level assignment = the parity target (DESIGN.md §2)
    rois = _convert_to_roi_format(boxes)
    want = torch.zeros(rois.shape[0], 32, 7, 7)
    for lvl, (f, s) in enumerate(zip(feats.values(), m.scales)):
        idx = torch.where(ref_levels.cpu() == lvl)[0]
        want[idx] = tv.ops.roi_align(f, rois[idx], 7, s, 2)
    vb.install()
    try:
        before = vb.launch_count()
        ours = m(fd, bd, shapes)
        used = vb.launch_count() - before
        assert used == 2, used                                       # ONE geometry launch + ONE gather launch for all four levels
        out2, levels = torch.ops.vision_b200.multiscale_roi_align(list(fd.values()), _convert_to_roi_format(bd), list(m.scales), 7, 7, 2,
                                                                  m.map_levels.k_min, m.map_levels.k_max, float(m.map_levels.s0),
                                                                  float(m.map_levels.lvl0), float(m.map_levels.eps))
        valid = (ref_levels >= 0) & (ref_levels < 4)                 # the inverted box has a NaN level in the reference (NaN.to(int64): no level matches, its row stays zero)
        bad = torch.where(valid & (levels.long() != ref_levels))[0]
        assert bad.numel() == 0, (bad.tolist()[:8], torch.cat(bd)[bad][:8].tolist(), levels[bad][:8].tolist(), ref_levels[bad][:8].tolist())
        assert torch.equal(ours, out2)
        np.testing.assert_allclose(npy(ours), want.numpy(), rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(npy(ours), npy(ref_cuda), rtol=1e-4, atol=1e-4)     # the CUDA reference is itself ~7e-5 from its CPU kernel
        # a shape the fused kernel does not cover (14x14 bins, the mask head) keeps working through the per-level loop
        m14 = MultiScaleRoIAlign(["0", "1", "2", "3"], 14, 2)
        o14 = m14(fd, bd, shapes)
    finally:
        vb.uninstall()
    np.testing.assert_allclose(npy(o14), npy(m14(fd, bd, shapes)), rtol=1e-4, atol=1e-4)
    # gradients of the fused op, per level, against the reference's autograd through its per-level loop
    fr = type(feats)((k, v.to(DEV).requires_grad_(True)) for k, v in feats.items())
    m(fr, bd, shapes).square().sum().backward()
    fo = [v.to(DEV).requires_grad_(True) for v in feats.values()]
    out, _ = torch.ops.vision_b200.multiscale_roi_align(fo, _convert_to_roi_format(bd), list(m.scales), 7, 7, 2, m.map_levels.k_min,
                                                        m.map_levels.k_max, float(m.map_levels.s0), float(m.map_levels.lvl0),
                                                        float(m.map_levels.eps))
    out.square().sum().backward()
    for a, b_ in zip(fo, fr.values()):
        np.testing.assert_allclose(npy(a.grad), npy(b_.grad), rtol=1e-3, atol=1e-3 * max(1.0, b_.grad.abs().max().item()))


# =============================== detection post-processing fused around NMS (SURVEY §8f3) ===============================
def _reference_tail(boxes, scores, labels, image_shape, score_thresh, inclusive, min_size, nms_thresh, topk):
    """The per-image tail of roi_heads.py:700-737 / rpn.py:273-298, verbatim tensor ops (reference kernels)."""
    from torchvision.ops import boxes as box_ops

    boxes = box_ops.clip_boxes_to_image(boxes, image_shape)
    inds = torch.where(scores >= score_thresh)[0] if inclusive else torch.where(scores > score_thresh)[0]
    boxes, scores, labels = boxes[inds], scores[inds], labels[inds]
    keep = box_ops.remove_small_boxes(boxes, min_size=min_size)
    boxes, scores, labels = boxes[keep], scores[keep], labels[keep]
    keep = box_ops.batched_nms(boxes, scores, labels, nms_thresh)[:topk]
    return boxes[keep], scores[keep], labels[keep]


@pytest.mark.parametrize("n,classes,topk,inclusive", [(90_000, 90, 100, False), (4000, 5, 1000, True), (300_000, 80, 2000, False), (50, 3, 10, True)])
def test_detection_postprocess_fused_bit_exact_vs_reference_tail(vb, n, classes, topk, inclusive):
    tv = pytest.importorskip("torchvision")
    from vision_b200 import detection

    assert not vb.installed()
    g = torch.Generator().manual_seed(n)
    xy = torch.rand(n, 2, generator=g) * torch.tensor([1100.0, 820.0]) - 20.0          # some boxes stick out of the 800 x 1088 image
    wh = torch.exp(torch.rand(n, 2, generator=g) * 6.0 - 3.0)                           # 0.05 .. 20 px .. 400 px: small boxes get removed
    boxes = torch.cat([xy, xy + wh], dim=1).to(DEV)
    scores = torch.rand(n, generator=g).to(DEV)
    scores[::17] = 0.05                                                                  # exactly at the threshold: '>' vs '>='
    labels = torch.randint(0, classes, (n,), generator=g).to(DEV)
    ref = _reference_tail(boxes, scores, labels, (800, 1088), 0.05, inclusive, 1e-2, 0.5, topk)
    before = vb.launch_count()
    ours = detection.detection_postprocess(boxes, scores, labels, (800, 1088), 0.05, inclusive, 1e-2, 0.5, topk)
    assert vb.launch_count() > before
    for a, b in zip(ours, ref):
        assert a.shape == b.shape and a.dtype == b.dtype and torch.equal(a, b)
    # nothing survives the filters / empty input
    none = detection.detection_postprocess(boxes[:100], scores[:100] * 0, labels[:100], (800, 1088), 0.5, False, 1e-2, 0.5, 10)
    assert none[0].shape == (0, 4) and none[1].shape == (0,) and none[2].dtype == torch.int64


# =============================== fused inference preprocessing (SURVEY §8f4) ===============================
@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32, torch.float16])
def test_classification_preset_fused_vs_reference(vb, dtype):
    """ImageClassification.forward (transforms/_presets.py:57-64) on CUDA tensors: the fused kernel against the reference's
    four passes.  uint8: the resized image is rounded to uint8 in the reference, so a value within ~1e-4 of a .5 tie may
    round differently (summation order) - those differ by exactly 1/255/std; everything else agrees to 1e-5."""
    tv = pytest.importorskip("torchvision")
    from torchvision.transforms._presets import ImageClassification

    assert not vb.installed()
    g = torch.Generator().manual_seed(3)
    for shape, crop, rs in (((4, 3, 375, 500), 224, 256), ((3, 600, 440), 224, 232), ((2, 1, 300, 300), 200, 256)):
        c = shape[-3]
        img = torch.randint(0, 256, shape, generator=g, dtype=torch.uint8)
        x = (img if dtype == torch.uint8 else (img.float() / 255).to(dtype)).to(DEV)
        preset = ImageClassification(crop_size=crop, resize_size=rs, mean=(0.485, 0.456, 0.406)[:c], std=(0.229, 0.224, 0.225)[:c])
        ref = preset(x)
        vb.install()
        try:
            before = vb.launch_count()
            ours = preset(x)
            assert vb.launch_count() == before + 1                     # ONE kernel
        finally:
            vb.uninstall()
        assert ours.shape == ref.shape and ours.dtype == torch.float32
        diff = (ours - ref).abs()
        if dtype == torch.uint8:
            step = 1.0 / 255 / 0.224
            off = diff > 1e-5
            assert float(off.float().mean()) < 2e-3 and float(diff.max()) <= step * 1.05
        elif dtype == torch.float16:
            assert float((diff > 1e-5).float().mean()) < 2e-3 and float(diff.max()) <= 2e-3 / 0.224      # one fp16 ulp of a value <= 1 before normalisation
        else:
            np.testing.assert_allclose(npy(ours), npy(ref), rtol=1e-5, atol=2e-5)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.float16])
def test_ps_roi_pool_forward_backward_vs_reference(vb, oracle, dtype):
    tv = pytest.importorskip("torchvision")
    assert not vb.installed()
    for shape, k, p, scale in [((2, 50, 30, 40), 500, 5, 0.5), ((1, 98, 40, 52), 1500, 7, 0.25), ((1, 18, 300, 400), 64, 3, 0.25)]:
        b, c, h, w = shape
        g = torch.Generator().manual_seed(k)
        x = torch.randn(*shape, generator=g)
        rois = _rois(k, b, h, w, scale, seed=k + 3)
        xd, rd = x.to(dtype).to(DEV), rois.to(dtype).to(DEV)
        o1, m1 = torch.ops.torchvision.ps_roi_pool(xd, rd, scale, p, p)
        o2, m2 = torch.ops.vision_b200.ps_roi_pool(xd, rd, scale, p, p)
        assert torch.equal(m1, m2)
        assert torch.equal(o1, o2), (shape, dtype, float((o1.float() - o2.float()).abs().max()))     # same adds in the same order
        if dtype == torch.float32:
            want, wm = oracle.ps_roi_pool(x.numpy(), rois.numpy(), p, scale)
            assert np.array_equal(npy(o2), want) and np.array_equal(npy(m2), wm)
        grad = (torch.randn(o1.shape, generator=g) * 0.25).to(dtype).to(DEV)
        args = (scale, p, p, b, c, h, w)
        # the integer bin windows depend on the dtype the box arithmetic runs in, so the ground truth is the reference in the
        # SAME dtype (its atomics only reorder the adds; in fp16 every add rounds to half, hence the loose bound there)
        truth = torch.ops.torchvision._ps_roi_pool_backward(grad, rd, m1, *args).double()
        ours = torch.ops.vision_b200._ps_roi_pool_backward(grad, rd, m1, *args)
        tol = {torch.float32: 1e-5, torch.float64: 1e-12, torch.float16: 3e-2}[dtype]
        np.testing.assert_allclose(ours.double().cpu().numpy(), truth.cpu().numpy(), rtol=tol, atol=tol * max(1.0, truth.abs().max().item()))
    vb.install()
    try:
        xr = torch.randn(1, 18, 20, 24, device=DEV, requires_grad=True)
        r = torch.tensor([[0, 2.0, 3.0, 60.0, 50.0], [0, 10.0, 10.0, 30.0, 70.0]], device=DEV)
        before = vb.launch_count()
        tv.ops.ps_roi_pool(xr, r, 3, 0.25).sum().backward()
        assert vb.launch_count() >= before + 2 and xr.grad.abs().sum().item() > 0
    finally:
        vb.uninstall()


# =============================== deform_conv2d backward (SURVEY §8f1) ===============================
def _dcn_args(batch, dtype, seed=0):
    # test/test_ops.py:1113-1167 get_fn_args: groups 2, offset groups 3, stride (2,1), pad (1,0), dil (2,1), kernel (3,2)
    g = torch.Generator().manual_seed(seed)
    cin, cout, ng, og, sh, sw, ph, pw, dh, dw, kh, kw, ih, iw = 6, 2, 2, 3, 2, 1, 1, 0, 2, 1, 3, 2, 5, 4
    oh = (ih + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1
    ow = (iw + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
    mk = lambda *s: torch.randn(*s, generator=g).to(dtype).to(DEV)
    x = torch.rand(batch, cin, ih, iw, generator=g).to(dtype).to(DEV)
    return (x, mk(cout, cin // ng, kh, kw), mk(batch, og * 2 * kh * kw, oh, ow), mk(batch, og * kh * kw, oh, ow), mk(cout),
            (sh, sw, ph, pw, dh, dw, ng, og))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_deform_conv2d_backward_vs_reference_cuda(vb, dtype):
    tv = pytest.importorskip("torchvision")
    from vision_b200 import workloads

    assert not vb.installed()
    cases = [_dcn_args(33, dtype), _dcn_args(1, dtype, seed=3)]
    x, off, w, b, m = workloads.cfg4_deform_conv2d(device=DEV, batch=2, c_in=64, c_out=128, hw=20, dtype=dtype)
    cases.append((x, w, off, m, b, (1, 1, 1, 1, 1, 1, 1, 1)))
    for (x, w, off, m, b, geo) in cases:
        for use_mask in (True, False):
            mm = m if use_mask else torch.zeros(x.shape[0], 1, device=DEV, dtype=dtype)
            out = torch.ops.torchvision.deform_conv2d(x, w, off, mm, b, *geo, use_mask)
            grad = torch.randn(out.shape, device=DEV, dtype=torch.float64).to(dtype) * 0.5
            truth = torch.ops.torchvision._deform_conv2d_backward(grad.double(), x.double(), w.double(), off.double(), mm.double(),
                                                                  b.double(), *geo, use_mask)
            ours = torch.ops.vision_b200._deform_conv2d_backward(grad, x, w, off, mm, b, *geo, use_mask)
            tol = 2e-5 if dtype == torch.float32 else 1e-10
            for name, a, t_ in zip(("input", "weight", "offset", "mask", "bias"), ours, truth):
                assert a.shape == t_.shape and a.dtype == dtype, name
                scale = max(1.0, t_.abs().max().item())
                np.testing.assert_allclose(a.double().cpu().numpy(), t_.cpu().numpy(), rtol=tol, atol=tol * scale, err_msg=name)


def test_deform_conv2d_gradcheck_and_installed_autograd(vb):
    """gradcheck in fp64 as test/test_ops.py:1236-1285 (fast_mode, nondet_tol for the atomics of grad_input); after install()
    torchvision.ops.deform_conv2d(...).backward() runs on our kernels."""
    tv = pytest.importorskip("torchvision")
    from torch.autograd import gradcheck

    assert not vb.installed()
    x, w, off, m, b, geo = _dcn_args(3, torch.float64, seed=1)
    sh, sw, ph, pw, dh, dw, ng, og = geo
    for t_ in (x, w, off, m, b):
        t_.requires_grad_(True)
    f = lambda x_, o_, m_, w_, b_: vb.ops.deform_conv2d(x_, o_, w_, b_, stride=(sh, sw), padding=(ph, pw), dilation=(dh, dw), mask=m_)
    assert gradcheck(f, (x, off, m, w, b), nondet_tol=1e-5, fast_mode=True)
    f2 = lambda x_, o_, w_, b_: vb.ops.deform_conv2d(x_, o_, w_, b_, stride=(sh, sw), padding=(ph, pw), dilation=(dh, dw), mask=None)
    assert gradcheck(f2, (x, off, w, b), nondet_tol=1e-5, fast_mode=True)
    # bf16 at a tensor-core shape: gradients flow and are finite, weight gradient close to an fp32 evaluation of the reference
    from vision_b200 import workloads
    xb, offb, wb, bb, mb = workloads.cfg4_deform_conv2d(device=DEV, batch=2, c_in=64, c_out=128, hw=16, dtype=torch.bfloat16)
    ref_in = [t_.float().requires_grad_(True) for t_ in (xb, offb, wb, bb, mb)]
    tv.ops.deform_conv2d(ref_in[0], ref_in[1], ref_in[2], ref_in[3], 1, 1, 1, ref_in[4]).square().mean().backward()
    vb.install()
    try:
        ours_in = [t_.clone().requires_grad_(True) for t_ in (xb, offb, wb, bb, mb)]
        before = vb.launch_count()
        tv.ops.deform_conv2d(ours_in[0], ours_in[1], ours_in[2], ours_in[3], 1, 1, 1, ours_in[4]).float().square().mean().backward()
        assert vb.launch_count() >= before + 3                       # forward + the two backward kernels
    finally:
        vb.uninstall()
    for a, r in zip(ours_in, ref_in):
        assert torch.isfinite(a.grad.float()).all()
        scale = r.grad.abs().max().item() + 1e-12
        assert (a.grad.float() - r.grad).abs().max().item() <= 5e-2 * scale


def test_deform_conv2d_packed_weight_cache_and_channels_last(vb):
    """The shim packs the weights once per (tensor, version) and hands a channels-last input to the tensor-core kernel
    without the staging pass: same bits as the plain call, fewer launches; an in-place weight update re-packs."""
    from vision_b200 import workloads

    for dtype in (torch.bfloat16, torch.float32):
        x, off, w, b, m = workloads.cfg4_deform_conv2d(device=DEV, batch=2, c_in=128, c_out=256, hw=24, dtype=dtype)
        base = vb.launch_count()
        first = vb.ops.deform_conv2d(x, off, w, b, 1, 1, 1, m)
        n_first = vb.launch_count() - base
        base = vb.launch_count()
        second = vb.ops.deform_conv2d(x, off, w, b, 1, 1, 1, m)
        n_second = vb.launch_count() - base
        assert torch.equal(first, second) and n_second == n_first - 1            # no pack_weights launch the second time
        xcl = x.contiguous(memory_format=torch.channels_last)
        base = vb.launch_count()
        third = vb.ops.deform_conv2d(xcl, off, w, b, 1, 1, 1, m)
        assert torch.equal(first, third) and vb.launch_count() - base == n_second - 1   # and no NCHW -> NHWC staging launch
        with torch.no_grad():
            w.mul_(0.5)                                                          # version bump: the cached image is stale
        fourth = vb.ops.deform_conv2d(x, off, w, b, 1, 1, 1, m)
        w2 = w.clone()
        assert torch.equal(fourth, vb.ops.deform_conv2d(x, off, w2, b, 1, 1, 1, m)) and not torch.equal(fourth, first)


def test_box_iou_rotated_vs_oracle_and_golden(vb, oracle):
    """Clipping-based kernel vs the oracle (itself bit-identical to the reference header, tests/test_oracle.py) and the fixture
    generated by the reference's own code.  The algorithms differ (clipping vs intersection points + hull), so the bound is a
    tolerance: 1e-5 absolute on the IoU, except pairs whose intersection is a sliver below the reference's own epsilons."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "box_iou_rotated.npz"))
    b1, b2 = torch.from_numpy(g["boxes1"]).to(DEV), torch.from_numpy(g["boxes2"]).to(DEV)
    before = vb.launch_count()
    got = vb.ops.box_iou_rotated(b1, b2)
    assert vb.launch_count() == before + 1 and got.shape == (257, 193) and got.dtype == torch.float32
    err = np.abs(npy(got) - g["ious"])
    assert err.max() <= 2e-5, (err.max(), np.unravel_index(err.argmax(), err.shape))
    np.testing.assert_allclose(npy(vb.ops.box_iou_rotated(torch.from_numpy(g["unit1"]).to(DEV), torch.from_numpy(g["unit2"]).to(DEV))),
                               g["unit_ious"], atol=1e-6)
    rng = np.random.default_rng(11)
    for n1, n2, span in ((1, 1, 10.0), (33, 65, 50.0), (1000, 777, 400.0)):
        c = rng.uniform(0, span, (n1 + n2, 2)); wh = np.exp(rng.uniform(0, 4.5, (n1 + n2, 2))); a = rng.uniform(-720, 720, (n1 + n2, 1))
        b = np.concatenate([c, wh, a], 1).astype(np.float32)
        want = oracle.box_iou_rotated(b[:n1], b[n1:])
        got = npy(vb.ops.box_iou_rotated(torch.from_numpy(b[:n1]).to(DEV), torch.from_numpy(b[n1:]).to(DEV)))
        assert np.abs(got - want).max() <= 2e-5
    assert vb.ops.box_iou_rotated(torch.zeros(0, 5, device=DEV), b2).shape == (0, 193)
    with pytest.raises(RuntimeError, match="Tensor\\[N, 5\\]"):
        vb.ops.box_iou_rotated(torch.zeros(3, 4, device=DEV), b2)


def test_batched_nms_graph_replay_matches_plain_launches(vb, oracle):
    """A repeating argument set is replayed as a CUDA graph from the third call on: same indices as the plain launches, also
    after the CONTENTS of the (same) buffers change; one launch is counted per replay."""
    from vision_b200 import workloads
    from test_gpu_parity import force_env

    b, s, i = [t_.to(DEV) for t_ in workloads.cfg3_batched_nms(n=60_000, seed=3)]
    with force_env("VB200_BNMS_GRAPH", "0"):
        plain = vb.ops.batched_nms(b, s, i, 0.5).clone()
    outs, counts = [], []
    for _ in range(4):
        before = vb.launch_count()
        outs.append(vb.ops.batched_nms(b, s, i, 0.5).clone())
        counts.append(vb.launch_count() - before)
    assert all(torch.equal(o, plain) for o in outs)
    assert counts[-1] <= 2 < counts[0]                   # graph replay: one graph launch instead of ~25 kernel launches
    b2, s2, i2 = workloads.cfg3_batched_nms(n=60_000, seed=4, clustered=True)
    b.copy_(b2.to(DEV)); s.copy_(s2.to(DEV)); i.copy_(i2.to(DEV))            # same addresses, new contents
    got = vb.ops.batched_nms(b, s, i, 0.5)
    want = oracle.batched_nms(b2.numpy(), s2.numpy(), i2.numpy(), 0.5, mode=oracle.NMS_MODE_CUDA, device_is_cuda=True)
    assert np.array_equal(npy(got), want)


# ---- resize fused with the all-gather of its output (peer stores): several destinations on ONE GPU --------------------------
@pytest.mark.gpu
def test_resize_gather_writes_every_destination(vb):
    """vision_b200::resize_gather stores each output pixel to all destinations (on a multi-GPU box: the same slot of every
    rank's gathered buffer).  Here the destinations are three slots of local buffers; each must equal the plain resize, and
    the bytes around the slots must stay untouched.  Streaming kernel (fp16 / uint8 bilinear-AA) and the copy fallback (bicubic)."""
    torch.manual_seed(0)
    for dtype, mode, aa, shape, size in ((torch.float16, 0, True, (5, 3, 270, 480), (64, 56)),
                                         (torch.uint8, 0, True, (2, 3, 300, 400), (40, 48)),
                                         (torch.float16, 1, True, (2, 3, 90, 120), (30, 40)),
                                         (torch.float32, 0, False, (2, 1, 33, 47), (20, 21))):
        x = (torch.rand(shape, device=DEV) * 255).to(dtype) if dtype == torch.uint8 else torch.rand(shape, device=DEV).to(dtype)
        want = torch.ops.vision_b200.resize(x, size[0], size[1], mode, aa)
        n = want.numel()
        bufs = [torch.full((n + 64,), 7, dtype=dtype, device=DEV) for _ in range(3)]
        ptrs = [b.data_ptr() + 32 * b.element_size() for b in bufs]
        torch.ops.vision_b200.resize_gather(x, ptrs, size[0], size[1], mode, aa)
        for b in bufs:
            assert torch.equal(b[32:32 + n].view(want.shape), want)
            assert bool((b[:32] == 7).all()) and bool((b[32 + n:] == 7).all())
    with pytest.raises(RuntimeError, match="1..8 destinations"):
        torch.ops.vision_b200.resize_gather(x, [], 4, 4, 0, True)


@pytest.mark.gpu
def test_roi_align_gather_writes_every_destination(vb):
    """vision_b200::roi_align_gather: the line kernel stores every bin to all destinations (peer slots on a multi-GPU box; three
    local buffers here); configurations the line kernel does not cover are computed once and copied."""
    from vision_b200 import workloads

    for (c, k, pool, dtype) in ((16, 300, 7, torch.float32), (8, 40, 5, torch.float32), (4, 30, 7, torch.float64)):
        x, rois, kw = workloads.cfg2_roi_align(seed=3, k=k, batch=2, channels=c, height=48, width=64)
        x, rois = x.to(DEV, dtype), rois.to(DEV, dtype)
        want = torch.ops.vision_b200.roi_align(x, rois, 0.25, pool, pool, 2, False)
        n = want.numel()
        bufs = [torch.full((n + 32,), -3.0, dtype=dtype, device=DEV) for _ in range(3)]
        ptrs = [b.data_ptr() + 16 * b.element_size() for b in bufs]
        torch.ops.vision_b200.roi_align_gather(x, rois, ptrs, 0, 0.25, pool, pool, 2, False)
        for b in bufs:
            assert torch.equal(b[16:16 + n].view(want.shape), want)
            assert bool((b[:16] == -3).all()) and bool((b[16 + n:] == -3).all())


@pytest.mark.gpu
def test_deform_conv2d_gather_writes_every_destination(vb):
    """vision_b200::deform_conv2d_gather: the wgmma epilogue stores each output element to all destinations (peer slots on a
    multi-GPU box; three local buffers here); shapes on the SIMT kernel are computed once and copied."""
    from vision_b200 import workloads

    for (cin, cout, hw, dtype) in ((64, 128, 16, torch.bfloat16), (8, 8, 9, torch.float32)):
        x, off, w, b, m = workloads.cfg4_deform_conv2d(seed=2, batch=2, c_in=cin, c_out=cout, hw=hw, dtype=dtype)
        x, off, w, b, m = [t.to(DEV) for t in (x, off, w, b, m)]
        want = torch.ops.vision_b200.deform_conv2d(x, w, off, m, b, 1, 1, 1, 1, 1, 1, 1, 1, True)
        n = want.numel()
        bufs = [torch.full((n + 128,), 5.0, dtype=dtype, device=DEV) for _ in range(3)]
        ptrs = [t.data_ptr() + 64 * t.element_size() for t in bufs]
        torch.ops.vision_b200.deform_conv2d_gather(x, w, off, m, b, ptrs, 1, 1, 1, 1, 1, 1, 1, 1, True)
        for t in bufs:
            assert torch.equal(t[64:64 + n].view(want.shape), want)
            assert bool((t[:64] == 5).all()) and bool((t[64 + n:] == 5).all())


@pytest.mark.gpu
def test_gather_helpers_without_a_process_group(vb):
    """sharded.resize_gather / roi_align_gather / deform_conv2d_gather with no peer buffer (one process, no group): the plain op."""
    from vision_b200 import sharded, workloads

    x = torch.rand(3, 3, 120, 200, device=DEV).half()
    got = sharded.resize_gather(x, [30, 40], None)
    assert torch.equal(got if isinstance(got, torch.Tensor) else got.materialize(), vb.transforms.resize_image(x, [30, 40]))
    f, rois, kw = workloads.cfg2_roi_align(seed=4, k=50, batch=1, channels=8, height=40, width=56)
    f, rois = f.to(DEV), rois.to(DEV)
    assert torch.equal(sharded.roi_align_gather(f, rois, None, **kw), vb.ops.roi_align(f, rois, **kw))
    xi, off, w, b, m = [t.to(DEV) for t in workloads.cfg4_deform_conv2d(seed=5, batch=1, c_in=8, c_out=8, hw=10, dtype=torch.float32)]
    assert torch.equal(sharded.deform_conv2d_gather(xi, off, w, b, None, 1, 1, 1, m), vb.ops.deform_conv2d(xi, off, w, b, 1, 1, 1, m))
