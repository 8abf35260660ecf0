"""deform_conv2d backward under torch.use_deterministic_algorithms: grad_input comes from the sorted-cell gather (written in
full, no atomics, bit-reproducible), checked against the reference's own backward run in float64 on the same values.

In deterministic mode torch fills at::empty with NaN, so a grad_input element the gather never writes shows up as NaN: every
case asserts isfinite.  The mode is entered with warn_only=True (still deterministic for the op): the shim's two dense GEMMs
are cuBLAS calls, which torch only warns about in this mode unless CUBLAS_WORKSPACE_CONFIG is set at process start."""
import contextlib
import ctypes
import warnings

import numpy as np
import pytest
import torch

DEV = "cuda"
NAMES = ("input", "weight", "offset", "mask", "bias")


@contextlib.contextmanager
def deterministic(warn_only=True):
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=warn_only)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", UserWarning)
            yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _ref_geometry(batch, dtype, seed=0):
    # test/test_ops.py:1113-1167 get_fn_args: groups 2, offset groups 3, stride (2,1), pad (1,0), dil (2,1), kernel (3,2)
    g = torch.Generator().manual_seed(seed)
    cin, cout, ng, og, sh, sw, ph, pw, dh, dw, kh, kw, ih, iw = 6, 2, 2, 3, 2, 1, 1, 0, 2, 1, 3, 2, 5, 4
    oh = (ih + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1
    ow = (iw + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
    mk = lambda *s: torch.randn(*s, generator=g).to(dtype).to(DEV)
    x = torch.rand(batch, cin, ih, iw, generator=g).to(dtype).to(DEV)
    return (x, mk(cout, cin // ng, kh, kw), mk(batch, og * 2 * kh * kw, oh, ow), mk(batch, og * kh * kw, oh, ow), mk(cout),
            (sh, sw, ph, pw, dh, dw, ng, og))


def _tc_shape(batch, dtype, seed=0):
    # 64 -> 128, 20 x 20, 3 x 3 (a tensor-core-sized layer)
    from vision_b200 import workloads

    x, off, w, b, m = workloads.cfg4_deform_conv2d(device=DEV, seed=seed, batch=batch, c_in=64, c_out=128, hw=20, dtype=dtype)
    return x, w, off, m, b, (1, 1, 1, 1, 1, 1, 1, 1)


def _custom(batch, cin, cout, hw, k, geo, dtype, offsets=None, seed=0):
    """geo = (sh, sw, ph, pw, dh, dw, groups, offset_groups); offsets(oh, ow) -> [batch, og*2*k*k, oh, ow] or None (random)."""
    g = torch.Generator().manual_seed(seed)
    sh, sw, ph, pw, dh, dw, ng, og = geo
    oh = (hw + 2 * ph - (dh * (k - 1) + 1)) // sh + 1
    ow = (hw + 2 * pw - (dw * (k - 1) + 1)) // sw + 1
    x = torch.randn(batch, cin, hw, hw, generator=g)
    w = torch.randn(cout, cin // ng, k, k, generator=g)
    off = offsets(oh, ow) if offsets is not None else torch.randn(batch, og * 2 * k * k, oh, ow, generator=g) * 1.5
    m = torch.rand(batch, og * k * k, oh, ow, generator=g)
    b = torch.randn(cout, generator=g)
    return tuple(t.to(dtype).to(DEV) for t in (x, w, off, m, b)) + (geo,)


def _grad_out(x, w, off, geo, dtype, seed=1):
    sh, sw, ph, pw, dh, dw, _, _ = geo
    kh, kw = w.shape[2], w.shape[3]
    oh = (x.shape[2] + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1
    ow = (x.shape[3] + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(x.shape[0], w.shape[0], oh, ow, generator=g, dtype=torch.float64) * 0.5).to(dtype).to(DEV)


def _mask_arg(x, m, use_mask):
    return m if use_mask else torch.zeros(x.shape[0], 1, device=DEV, dtype=x.dtype)


def _ours(grad, x, w, off, m, b, geo, use_mask):
    return torch.ops.vision_b200._deform_conv2d_backward(grad, x, w, off, _mask_arg(x, m, use_mask), b, *geo, use_mask)


def _truth(grad, x, w, off, m, b, geo, use_mask):
    mm = _mask_arg(x, m, use_mask)
    return torch.ops.torchvision._deform_conv2d_backward(grad.double(), x.double(), w.double(), off.double(), mm.double(), b.double(),
                                                         *geo, use_mask)


def _check_vs_truth(ours, truth, tol):
    for name, a, t_ in zip(NAMES, ours, truth):
        assert a.shape == t_.shape, name
        assert torch.isfinite(a).all(), name
        scale = max(1.0, t_.abs().max().item())
        np.testing.assert_allclose(a.double().cpu().numpy(), t_.cpu().numpy(), rtol=tol, atol=tol * scale, err_msg=name)


# ---------------------------------------------------------------- 1. parity, fp32 / fp64
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_parity_vs_reference_fp64(vb, dtype):
    pytest.importorskip("torchvision")
    tol = 2e-5 if dtype == torch.float32 else 1e-10
    for case in (_ref_geometry(33, dtype), _ref_geometry(1, dtype, seed=3), _tc_shape(2, dtype)):
        x, w, off, m, b, geo = case
        grad = _grad_out(x, w, off, geo, dtype)
        for use_mask in (True, False):
            truth = _truth(grad, x, w, off, m, b, geo, use_mask)
            with deterministic():
                ours = _ours(grad, x, w, off, m, b, geo, use_mask)
            _check_vs_truth(ours, truth, tol)


# ---------------------------------------------------------------- 2. 16-bit
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_16bit_grad_input_no_worse_than_atomics(vb, dtype):
    """One fp32 accumulator rounded once: the gathered grad_input is at least as close to the fp64 truth as the atomic
    scatter, whose every add rounds to 16 bits."""
    pytest.importorskip("torchvision")
    x, w, off, m, b, geo = _tc_shape(2, dtype)
    grad = _grad_out(x, w, off, geo, dtype)
    truth = _truth(grad, x, w, off, m, b, geo, True)[0]
    atomic = _ours(grad, x, w, off, m, b, geo, True)[0]
    with deterministic():
        ours = _ours(grad, x, w, off, m, b, geo, True)
    assert all(torch.isfinite(t_.float()).all() for t_ in ours)
    err_det = (ours[0].double() - truth).abs().max().item()
    err_atomic = (atomic.double() - truth).abs().max().item()
    assert err_det <= err_atomic, (err_det, err_atomic)
    assert err_det <= 1e-2 * max(1.0, truth.abs().max().item())


# ---------------------------------------------------------------- 3. reproducibility
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.float16, torch.bfloat16])
def test_two_calls_bit_identical(vb, dtype):
    cases = [_tc_shape(3, dtype)]
    if dtype in (torch.float32, torch.float64):
        cases.append(_ref_geometry(33, dtype))
    for x, w, off, m, b, geo in cases:
        grad = _grad_out(x, w, off, geo, dtype)
        for use_mask in (True, False):
            with deterministic():
                first = _ours(grad, x, w, off, m, b, geo, use_mask)
                second = _ours(grad, x, w, off, m, b, geo, use_mask)
            for name, a, c in zip(NAMES, first, second):
                assert torch.equal(a, c), name
            assert torch.isfinite(first[0].float()).all()


@pytest.mark.gpu
def test_collision_every_sample_in_one_cell(vb):
    """All 9 x 256 samples of an image land in the cell (7, 9): 2304 terms into each of four pixels per channel.  Identical
    over three calls; within n_terms * 2^-24 of the fp64 truth, relative to the sum of the terms' magnitudes."""
    pytest.importorskip("torchvision")
    k, hw = 3, 16
    ty, tx = 7.3, 9.6

    def offsets(oh, ow):
        oy = torch.arange(oh, dtype=torch.float64).view(1, 1, oh, 1)
        ox = torch.arange(ow, dtype=torch.float64).view(1, 1, 1, ow)
        taps = torch.arange(k * k)
        i = (taps // k).double().view(1, -1, 1, 1)
        j = (taps % k).double().view(1, -1, 1, 1)
        dy = (ty - (oy - 1 + i)).expand(1, k * k, oh, ow)
        dx = (tx - (ox - 1 + j)).expand(1, k * k, oh, ow)
        return torch.stack([dy, dx], 2).reshape(1, 2 * k * k, oh, ow).float()

    x, w, off, m, b, geo = _custom(1, 4, 4, hw, k, (1, 1, 1, 1, 1, 1, 1, 1), torch.float32, offsets=offsets)
    grad = _grad_out(x, w, off, geo, torch.float32)
    with deterministic():
        runs = [_ours(grad, x, w, off, m, b, geo, True)[0] for _ in range(3)]
    assert torch.equal(runs[0], runs[1]) and torch.equal(runs[0], runs[2])
    gi = runs[0]
    assert torch.isfinite(gi).all()
    assert ((gi != 0).sum(dim=(2, 3)) <= 4).all()                 # only the cell's four pixels receive anything
    truth = _truth(grad, x, w, off, m, b, geo, True)[0]
    magnitude = _truth(grad.abs(), x, w.abs(), off, m.abs(), b, geo, True)[0]      # >= the sum of |term| per element
    n_terms = k * k * hw * hw
    bound = n_terms * 2.0 ** -24 * magnitude + 1e-30
    assert ((gi.double() - truth).abs() <= bound).all()
    assert truth.abs().max().item() > 0


# ---------------------------------------------------------------- 4. batch invariance
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float64])
def test_image_gradients_independent_of_the_batch(vb, dtype):
    case = _tc_shape(4, dtype) if dtype != torch.float64 else _ref_geometry(5, dtype)
    x, w, off, m, b, geo = case
    grad = _grad_out(x, w, off, geo, dtype)
    with deterministic():
        full = _ours(grad, x, w, off, m, b, geo, True)
        for i in range(x.shape[0]):
            s = slice(i, i + 1)
            one = _ours(grad[s].clone(), x[s].clone(), w, off[s].clone(), m[s].clone(), b, geo, True)
            for k_ in (0, 2, 3):                                     # grad_input, grad_offset, grad_mask
                assert torch.equal(full[k_][s], one[k_]), (i, NAMES[k_])


# ---------------------------------------------------------------- 5. geometry edges
def _positions(y, x):
    """offsets of a 1 x 1, stride 1, pad 0 kernel that put the sample of output pixel (oy, ox) at (y[oy, ox], x[oy, ox])."""
    oh, ow = y.shape
    gy = torch.arange(oh, dtype=torch.float64).view(oh, 1)
    gx = torch.arange(ow, dtype=torch.float64).view(1, ow)
    return torch.stack([y - gy, x - gx], 0).view(1, 2, oh, ow).float()


@pytest.mark.gpu
def test_geometry_edges(vb):
    pytest.importorskip("torchvision")
    hw = 12
    gen = torch.Generator().manual_seed(5)
    one = (1, 1, 0, 0, 1, 1, 1, 1)
    # samples partly outside: y, x in (-1, 0) and (H-1, H) among the rest
    edge = torch.tensor([-0.75, -0.25, 11.25, 11.8])
    ys = torch.rand(hw, hw, generator=gen, dtype=torch.float64) * (hw + 1) - 1
    xs = torch.rand(hw, hw, generator=gen, dtype=torch.float64) * (hw + 1) - 1
    ys[0, :4], xs[1, :4], ys[2, :4], xs[2, :4] = edge, edge, edge, edge.flip(0)
    cases = [
        ("partly outside", _custom(1, 3, 2, hw, 1, one, torch.float32, offsets=lambda oh, ow: _positions(ys, xs))),
        ("zero offsets", _custom(2, 3, 2, hw, 3, (1, 1, 1, 1, 1, 1, 1, 1), torch.float32,
                                 offsets=lambda oh, ow: torch.zeros(2, 18, oh, ow))),
        ("1x1", _custom(2, 5, 3, hw, 1, one, torch.float32)),
        ("dilated 5x5", _custom(2, 4, 4, hw, 5, (1, 1, 4, 4, 2, 2, 1, 1), torch.float32)),
        ("offset groups 4, groups 2", _custom(2, 8, 6, hw, 3, (2, 1, 1, 0, 1, 2, 2, 4), torch.float32)),
    ]
    for name, (x, w, off, m, b, geo) in cases:
        grad = _grad_out(x, w, off, geo, torch.float32)
        for use_mask in (True, False):
            truth = _truth(grad, x, w, off, m, b, geo, use_mask)
            with deterministic():
                ours = _ours(grad, x, w, off, m, b, geo, use_mask)
            try:
                _check_vs_truth(ours, truth, 2e-5)
            except AssertionError as e:
                raise AssertionError(f"{name}, use_mask={use_mask}: {e}") from None
    # every sample outside the image: grad_input is exactly 0 (written, not left NaN)
    x, w, off, m, b, geo = _custom(2, 3, 2, hw, 3, (1, 1, 1, 1, 1, 1, 1, 1), torch.float32,
                                   offsets=lambda oh, ow: torch.full((2, 18, oh, ow), -30.0))
    grad = _grad_out(x, w, off, geo, torch.float32)
    with deterministic():
        gi = _ours(grad, x, w, off, m, b, geo, True)[0]
    assert torch.equal(gi, torch.zeros_like(gi))


# ---------------------------------------------------------------- 6. gradcheck without slack
@pytest.mark.gpu
def test_gradcheck_deterministic_no_nondet_tol(vb):
    from torch.autograd import gradcheck

    x, w, off, m, b, geo = _ref_geometry(3, torch.float64, seed=1)
    sh, sw, ph, pw, dh, dw, ng, og = geo
    for t_ in (x, w, off, m, b):
        t_.requires_grad_(True)
    f = lambda x_, o_, m_, w_, b_: vb.ops.deform_conv2d(x_, o_, w_, b_, stride=(sh, sw), padding=(ph, pw), dilation=(dh, dw), mask=m_)
    f2 = lambda x_, o_, w_, b_: vb.ops.deform_conv2d(x_, o_, w_, b_, stride=(sh, sw), padding=(ph, pw), dilation=(dh, dw), mask=None)
    with deterministic():
        assert gradcheck(f, (x, off, m, w, b), nondet_tol=0.0, fast_mode=True)
        assert gradcheck(f2, (x, off, w, b), nondet_tol=0.0, fast_mode=True)


# ---------------------------------------------------------------- 7. through torchvision
@pytest.mark.gpu
def test_installed_torchvision_backward_is_reproducible(vb):
    tv = pytest.importorskip("torchvision")
    from torch.profiler import ProfilerActivity, profile

    x0, w0, off0, m0, b0, _ = _tc_shape(2, torch.float32)

    def run():
        ins = [t_.clone().requires_grad_(True) for t_ in (x0, off0, w0, b0, m0)]
        tv.ops.deform_conv2d(ins[0], ins[1], ins[2], ins[3], 1, 1, 1, ins[4]).square().mean().backward()
        return [t_.grad for t_ in ins]

    assert not vb.installed()
    vb.install()
    try:
        with deterministic():
            before = vb.launch_count()
            first = run()
            assert vb.launch_count() >= before + 7          # forward + grad_offset/mask + bin, sort, table, records, gather
            second = run()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run()
                torch.cuda.synchronize()
    finally:
        vb.uninstall()
    for a, c in zip(first, second):
        assert torch.isfinite(a).all() and torch.equal(a, c)
    assert any("dcn_grad_input_gather_kernel" in e.key for e in prof.key_averages())
    # the reference's backward refuses this mode
    ins = [t_.clone().requires_grad_(True) for t_ in (x0, off0, w0, b0, m0)]
    out = tv.ops.deform_conv2d(ins[0], ins[1], ins[2], ins[3], 1, 1, 1, ins[4]).square().mean()
    with pytest.raises(RuntimeError):
        with deterministic(warn_only=False):
            out.backward()


# ---------------------------------------------------------------- 8. workspace query (no GPU)
def test_backward_inputs_workspace_query_needs_no_gpu():
    from vision_b200 import _lib

    lib = _lib.core()
    q = lib.vb200_deform_conv2d_backward_inputs_workspace_bytes
    f32, f64 = 0, 3

    def ws(dtype=f32, n=1, c=8, h=16, w=16, k=3, og=1):
        return q(dtype, n, c, h, w, k, k, 1, 1, 1, 1, 1, 1, og)

    assert ws(n=0) == 0 and ws(c=0) == 0 and ws(h=0) == 0
    assert ws(og=3) == 0                                        # 8 channels do not split into 3 offset groups
    assert 0 < ws(n=1) < ws(n=2) < ws(n=8)
    assert ws(h=16) < ws(h=32) and ws(k=3) < ws(k=5) and ws(og=1) < ws(og=2)
    assert ws(dtype=f64) > ws(dtype=f32)
    # at least the keys, values (both double-buffered) and one record per sample
    n_samples = 2 * 9 * 64 * 64
    assert ws(n=2, h=64, w=64) >= n_samples * (16 + 24)
