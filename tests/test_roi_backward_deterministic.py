"""Backward of roi_align / roi_pool / ps_roi_align / ps_roi_pool under torch.use_deterministic_algorithms: grad_input comes
from the row-owning plane kernels (written in full, no global atomics, bit-reproducible) for fp32, fp64 and fp16, every
sampling ratio and planes larger than shared memory (row-tiled), checked against the reference's own backward run in fp64.

In deterministic mode torch fills at::empty with NaN, so a grad_input element no kernel writes shows up as NaN: every case
asserts isfinite."""
import contextlib

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
DTYPES = (torch.float32, torch.float64, torch.float16)


@contextlib.contextmanager
def deterministic(warn_only=True):
    """Deterministic mode; strict (warn_only=False) turns every fall-back to a non-deterministic kernel into an error."""
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=warn_only)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _rois(k, b, h, w, scale, g, quantum=None):
    """RoIs in input coordinates (feature plane h x w at `scale`): a third tiny, a third reaching past the border, the
    rest anywhere (so some span the row tiles of a large plane).  quantum: corners on multiples of it in feature pixels."""
    fh, fw = h / scale, w / scale
    x1 = torch.rand(k, generator=g) * fw * 1.05 - 0.05 * fw
    y1 = torch.rand(k, generator=g) * fh * 1.05 - 0.05 * fh
    size = torch.rand(k, 2, generator=g) * torch.tensor([fw, fh]) * 0.6
    kind = torch.arange(k) % 3
    size[kind == 0] *= 0.02                                  # tiny: smaller than a bin
    size[kind == 1] += torch.tensor([fw, fh]) * 0.3          # large, mostly past the border
    x2, y2 = x1 + size[:, 0], y1 + size[:, 1]
    box = torch.stack([x1, y1, x2, y2], 1)
    if quantum is not None:
        q = quantum / scale
        box = (box / q).round() * q
    return torch.cat([torch.randint(0, b, (k, 1), generator=g).double(), box.double()], 1)


def _case(op, dtype, h, w, sr, aligned=False, seed=0, p=(7, 7)):
    """(call(grad) -> grad_input via vision_b200, truth in fp64 via the reference, the reference's own backward in dtype, grad)."""
    g = torch.Generator().manual_seed(seed)
    b, k, scale = 2, 60, 0.25
    ph, pw = p
    c = 3 if op in ("roi_align", "roi_pool") else 2 * ph * pw
    rois = _rois(k, b, h, w, scale, g, quantum=ph if op == "ps_roi_pool" else None)
    x = torch.randn(b, c, h, w, generator=g, dtype=torch.float64)
    tv = torch.ops.torchvision
    ours = torch.ops.vision_b200
    rd = rois.to(dtype).to(DEV)
    rd64 = rd.double()
    if op == "roi_align":
        grad = (torch.randn(k, c, ph, pw, generator=g, dtype=torch.float64) * 0.25).to(dtype).to(DEV)
        args = (scale, ph, pw, b, c, h, w, sr, aligned)
        return (lambda gr: ours._roi_align_backward(gr, rd, *args), tv._roi_align_backward(grad.double(), rd64, *args),
                lambda: tv._roi_align_backward(grad, rd, *args), grad)
    if op == "ps_roi_align":
        xd = x.to(dtype).to(DEV)
        out, mapping = tv.ps_roi_align(xd, rd, scale, ph, pw, sr)
        grad = (torch.randn(out.shape, generator=g, dtype=torch.float64) * 0.25).to(dtype).to(DEV)
        args = (scale, ph, pw, sr, b, c, h, w)
        return (lambda gr: ours._ps_roi_align_backward(gr, rd, mapping, *args),
                tv._ps_roi_align_backward(grad.double(), rd64, mapping, *args),
                lambda: tv._ps_roi_align_backward(grad, rd, mapping, *args), grad)
    if op == "roi_pool":
        x[:, :, ::2, ::2] = 1.5                                  # ties: neighbouring bins share their argmax
        out, am = tv.roi_pool(x.to(dtype).to(DEV), rd, scale, ph, pw)
        grad = (torch.randn(out.shape, generator=g, dtype=torch.float64) * 0.25).to(dtype).to(DEV)
        args = (scale, ph, pw, b, c, h, w)
        return (lambda gr: ours._roi_pool_backward(gr, rd, am, *args), tv._roi_pool_backward(grad.double(), rd64, am, *args),
                lambda: tv._roi_pool_backward(grad, rd, am, *args), grad)
    # ps_roi_pool: corners on whole bins, so the bin windows come out the same in fp16, fp32 and fp64
    out, mapping = tv.ps_roi_pool(x.to(dtype).to(DEV), rd, scale, ph, pw)
    grad = (torch.randn(out.shape, generator=g, dtype=torch.float64) * 0.25).to(dtype).to(DEV)
    args = (scale, ph, pw, b, c, h, w)
    return (lambda gr: ours._ps_roi_pool_backward(gr, rd, mapping, *args),
            tv._ps_roi_pool_backward(grad.double(), rd64, mapping, *args),
            lambda: tv._ps_roi_pool_backward(grad, rd, mapping, *args), grad)


def _check(vb, op, dtype, h, w, sr, aligned=False, p=(7, 7)):
    call, truth, ref_call, grad = _case(op, dtype, h, w, sr, aligned, seed=h + w + abs(sr) + 7 * aligned, p=p)
    before = vb.launch_count()
    with deterministic(warn_only=False):            # strict: a fall-back to the atomic kernels would raise
        first = call(grad)
        again = call(grad)
    assert vb.launch_count() > before
    assert first.dtype == dtype and first.shape == truth.shape
    assert torch.isfinite(first).all(), "grad_input not written in full"
    assert torch.equal(first, again), "not bit-reproducible"
    scale = truth.abs().max().item() + 1e-12
    err = (first.double() - truth).abs().max().item()
    if dtype == torch.float32:
        # the bound of the fp32 plane-path tests (test_gpu_round2.py), applied, where RoI corners of a few hundred pixels put the
        # reference's own fp32 backward further from the fp64 truth (coordinate rounding), on top of that kernel's error
        err_ref = (ref_call().double() - truth).abs().max().item()
        assert err <= err_ref + 1e-5 * (1 + scale), (err, err_ref, scale)
    elif dtype == torch.float64:
        assert err <= 1e-10 * max(1.0, scale), (err, scale)
    else:
        # fp16: no worse than 1.5x the reference's own fp16 backward (half atomics, half coordinates), against the same
        # fp64 truth; floor: two half ulps of the largest value
        err_ref = (ref_call().double() - truth).abs().max().item()
        assert err <= max(1.5 * err_ref, 2.0 ** -10 * scale), (err, err_ref, scale)


# a plane that fits shared memory and one that does not (tiled): 192 x 336 is FPN P2 of an 800 x 1333 image padded to 768 x
# 1344; an fp16 plane tiles with fp32 accumulators, fp64 at 200 x 272 already needs two tiles
def _planes(dtype):
    return [(50, 68), (200, 272) if dtype == torch.float64 else (192, 336)]


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("sr", [2, 0, -1])
@pytest.mark.parametrize("op,aligned", [("roi_align", False), ("roi_align", True), ("ps_roi_align", False)])
def test_align_ops_deterministic(vb, op, aligned, sr, dtype):
    pytest.importorskip("torchvision")
    for h, w in _planes(dtype):
        _check(vb, op, dtype, h, w, sr, aligned)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("op", ["roi_pool", "ps_roi_pool"])
def test_pool_ops_deterministic(vb, op, dtype):
    pytest.importorskip("torchvision")
    for h, w in _planes(dtype):
        _check(vb, op, dtype, h, w, 1, p=(7, 7) if op == "roi_pool" else (3, 3))


def test_roi_align_14x14_tiled(vb):
    """The table kernel's multi-chunk variant (28 y samples, 56 x taps, 196 bins) on a tiled plane."""
    pytest.importorskip("torchvision")
    for dtype in DTYPES:
        _check(vb, "roi_align", dtype, 192, 336, 2, p=(14, 14))


@pytest.mark.parametrize("kind", ["roi_align7", "roi_align14", "roi_pool", "ps_roi_align"])
def test_tiling_does_not_change_bits(vb, kind):
    """fp32: RoIs in rows 40..150, columns 0..80 of a 192 x 336 plane (two row tiles of 96, so they cross the tile
    boundary) give the same bits as on a 160 x 96 plane that fits in one piece, and zero elsewhere.  160 x 96 keeps every
    sample off the small plane's border clamp."""
    tv = pytest.importorskip("torchvision")
    g = torch.Generator().manual_seed(3)
    b, k = 2, 200
    p = 14 if kind == "roi_align14" else 7
    c = 2 * p * p if kind == "ps_roi_align" else 4
    x1 = torch.rand(k, generator=g) * 70
    y1 = 40 + torch.rand(k, generator=g) * 100
    x2 = torch.minimum(x1 + torch.rand(k, generator=g) * 40, torch.tensor(80.0))
    y2 = torch.minimum(y1 + torch.rand(k, generator=g) * 60, torch.tensor(150.0))
    rois = torch.cat([torch.randint(0, b, (k, 1), generator=g).float(), torch.stack([x1, y1, x2, y2], 1)], 1).to(DEV)
    ops = torch.ops.vision_b200
    small_hw, big_hw = (160, 96), (192, 336)
    with deterministic():
        if kind.startswith("roi_align"):
            grad = torch.randn(k, c, p, p, generator=g).to(DEV)
            run = lambda h, w: ops._roi_align_backward(grad, rois, 1.0, p, p, b, c, h, w, 2, True)
            small, big = run(*small_hw), run(*big_hw)
        elif kind == "ps_roi_align":
            cout = c // (p * p)
            grad = torch.randn(k, cout, p, p, generator=g).to(DEV)
            mapping = torch.zeros(k, cout, p, p, dtype=torch.int32, device=DEV)
            run = lambda h, w: ops._ps_roi_align_backward(grad, rois, mapping, 1.0, p, p, 2, b, c, h, w)
            small, big = run(*small_hw), run(*big_hw)
        else:
            x = torch.randn(b, c, *small_hw, generator=g).to(DEV)
            out, am = torch.ops.torchvision.roi_pool(x, rois, 1.0, p, p)
            grad = torch.randn(out.shape, generator=g).to(DEV)
            am_big = torch.where(am >= 0, am // small_hw[1] * big_hw[1] + am % small_hw[1], am)
            small = ops._roi_pool_backward(grad, rois, am, 1.0, p, p, b, c, *small_hw)
            big = ops._roi_pool_backward(grad, rois, am_big, 1.0, p, p, b, c, *big_hw)
    assert small.abs().sum() > 0
    assert torch.equal(big[:, :, :small_hw[0], :small_hw[1]], small)
    rest = big.clone()
    rest[:, :, :small_hw[0], :small_hw[1]] = 0
    assert torch.equal(rest, torch.zeros_like(rest))


def _gradcheck_cases(tv_ops, vb_ops):
    x = torch.rand(1, 2 * 2 * 2, 10, 10, dtype=torch.float64, device=DEV, requires_grad=True)
    rois = torch.tensor([[0, 0, 0, 9, 9], [0, 0, 5, 4, 9], [0, 5, 5, 9, 9], [0, 1.5, 2.25, 7.5, 8.75]], dtype=torch.float64, device=DEV)
    for ops in (tv_ops, vb_ops):
        for sr in (2, -1):
            for aligned in (False, True):
                yield f"roi_align sr={sr} aligned={aligned}", lambda t, o=ops, s=sr, a=aligned: o.roi_align(t, rois, 5, 0.5, s, a), x
            yield f"ps_roi_align sr={sr}", lambda t, o=ops, s=sr: o.ps_roi_align(t, rois, 2, 0.5, s), x
        yield "roi_pool", lambda t, o=ops: o.roi_pool(t, rois, 5, 0.5), x
        yield "ps_roi_pool", lambda t, o=ops: o.ps_roi_pool(t, rois, 2, 0.5), x


def test_gradcheck_fp64_nondet_tol_zero(vb):
    """fp64 gradcheck with nondet_tol=0 in deterministic mode, through vision_b200.ops and through torchvision.ops after
    install() (test/test_ops.py's gradchecks)."""
    tv = pytest.importorskip("torchvision")
    from torch.autograd import gradcheck

    vb.install()
    try:
        before = vb.launch_count()
        with deterministic(warn_only=False):
            for name, fn, x in _gradcheck_cases(tv.ops, vb.ops):
                assert gradcheck(fn, (x,), nondet_tol=0.0, fast_mode=False), name
        assert vb.launch_count() > before
    finally:
        vb.uninstall()


def test_multiscale_roi_align_strict_mode(vb):
    """The user scenario: Faster / Mask R-CNN box and mask heads on FPN features of a padded 800 x 1344 batch of 2, forward
    and backward in strict deterministic mode (warn_only=False); two runs give the same gradient bits on every level."""
    tv = pytest.importorskip("torchvision")
    from collections import OrderedDict

    g = torch.Generator().manual_seed(0)
    feats = OrderedDict((str(i), torch.randn(2, 256, 800 // s, 1344 // s, generator=g).to(DEV)) for i, s in enumerate((4, 8, 16, 32)))
    sizes = [(800, 1344)] * 2
    boxes = []
    for _ in range(2):
        wh = torch.exp(torch.rand(500, 2, generator=g) * 4.0 + 2.5)
        xy = torch.rand(500, 2, generator=g) * torch.tensor([1344.0, 800.0]) * 0.9
        boxes.append(torch.cat([xy, torch.minimum(xy + wh, torch.tensor([1344.0, 800.0]))], 1).to(DEV))
    vb.install()
    try:
        for out in (7, 14):
            pool = tv.ops.MultiScaleRoIAlign(["0", "1", "2", "3"], out, 2)
            grads = []
            for _ in range(2):
                leaves = OrderedDict((k, v.clone().requires_grad_(True)) for k, v in feats.items())
                with deterministic(warn_only=False):
                    y = pool(leaves, boxes, sizes)
                    y.backward(torch.ones_like(y))
                grads.append([leaves[k].grad for k in leaves])
            for a, b in zip(*grads):
                assert torch.isfinite(a).all() and torch.equal(a, b)
            assert grads[0][0].abs().sum() > 0
    finally:
        vb.uninstall()


@pytest.mark.parametrize("dtype,width", [(torch.float32, 60000), (torch.float64, 30000)], ids=["fp32", "fp64"])
def test_row_too_wide_raises_in_strict_mode(vb, dtype, width):
    """A grad_input row that does not fit in shared memory is the one shape the deterministic kernels do not take: strict
    mode raises with the op's name, as the reference does for every shape."""
    rois = torch.tensor([[0, 0, 0, 8, 3]], dtype=dtype, device=DEV)
    ops = torch.ops.vision_b200
    calls = {
        "roi_align_backward": lambda: ops._roi_align_backward(torch.ones(1, 1, 2, 2, dtype=dtype, device=DEV), rois, 1.0, 2, 2, 1, 1, 4,
                                                              width, 2, False),
        "roi_pool_backward": lambda: ops._roi_pool_backward(torch.ones(1, 1, 2, 2, dtype=dtype, device=DEV), rois,
                                                            torch.zeros(1, 1, 2, 2, dtype=torch.int32, device=DEV), 1.0, 2, 2, 1, 1, 4, width),
        "ps_roi_align_backward": lambda: ops._ps_roi_align_backward(torch.ones(1, 1, 2, 2, dtype=dtype, device=DEV), rois,
                                                                    torch.zeros(1, 1, 2, 2, dtype=torch.int32, device=DEV), 1.0, 2, 2, 2,
                                                                    1, 4, 4, width),
        "ps_roi_pool_backward": lambda: ops._ps_roi_pool_backward(torch.ones(1, 1, 2, 2, dtype=dtype, device=DEV), rois,
                                                                  torch.zeros(1, 1, 2, 2, dtype=torch.int32, device=DEV), 1.0, 2, 2, 1, 4,
                                                                  4, width),
    }
    for name, call in calls.items():
        with deterministic(warn_only=False):
            with pytest.raises(RuntimeError, match=name):
                call()
        with deterministic(warn_only=True):       # torch warns (on stderr) and the atomic kernel runs
            got = call()
        assert torch.isfinite(got).all() and got.abs().sum() > 0
