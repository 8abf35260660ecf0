"""CPU suite: FCOS.compute_loss is rebound by install() and restored by uninstall(); inputs the FCOS matching kernel does not
cover keep running the reference body; the level-boundary rule follows the reference's own slicing; the fake op gives the
reference's shapes."""
import ctypes
import types

import pytest
import torch

tv = pytest.importorskip("torchvision")
from torchvision.models.detection import fcos  # noqa: E402

import vision_b200  # noqa: E402
from vision_b200 import _lib, detection as det  # noqa: E402


class _SeenAsCuda(torch.Tensor):
    """A CPU tensor the coverage predicate takes for a CUDA one, so that each case below is refused for its own reason
    and the reference body can still run here."""

    @property
    def is_cuda(self):
        return True


def _cuda(t):
    return t.as_subclass(_SeenAsCuda)


def _anchors(side=64, strides=(8, 16, 32, 64, 128)):
    """FCOS's anchors of a side x side image: one stride-sized box per location and level (anchor_utils.py)."""
    per_level = []
    for s in strides:
        n = -(-side // s)
        c = torch.arange(n, dtype=torch.float32) * s
        y, x = torch.meshgrid(c, c, indexing="ij")
        xy = torch.stack([x.reshape(-1), y.reshape(-1)], 1)
        per_level.append(torch.cat([xy - s / 2, xy + s / 2], 1))
    return torch.cat(per_level), [p.shape[0] for p in per_level]


def _gt(n, seed, dtype=torch.float32):
    gen = torch.Generator().manual_seed(seed)
    xy = torch.rand(n, 2, generator=gen) * 40
    return torch.cat([xy, xy + torch.rand(n, 2, generator=gen) * 30 + 4], 1).to(dtype)


def _owner(radius=1.5):
    """A stand-in FCOS: compute_loss reads only these attributes; the head returns the matched indices."""
    head = types.SimpleNamespace(compute_loss=lambda targets, outputs, anchors, matched: matched)
    return types.SimpleNamespace(center_sampling_radius=radius, head=head)


def _call(owner, gts, anchors, levels):
    return fcos.FCOS.compute_loss(owner, [{"boxes": g} for g in gts], {}, anchors, levels)


def _same(a, b):
    if isinstance(a, (list, tuple)):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            _same(x, y)
        return
    assert a.dtype == b.dtype and a.shape == b.shape and a.stride() == b.stride()
    assert torch.equal(torch.as_tensor(a), torch.as_tensor(b))


def _refuse(*a, **k):
    raise AssertionError("the fused path must not be taken for these inputs")


def test_install_rebinds_and_restores_fcos_compute_loss():
    orig = fcos.FCOS.compute_loss
    vision_b200.install()
    try:
        assert fcos.FCOS.compute_loss is not orig and fcos.FCOS.compute_loss.__wrapped__ is orig
        from vision_b200 import _install

        assert _install._state["matching"][(fcos.FCOS, "compute_loss")] is orig
    finally:
        vision_b200.uninstall()
    assert fcos.FCOS.compute_loss is orig


def _cases():
    a, levels = _anchors()
    gts, anchors = [_gt(3, 0), _gt(2, 1)], [a, a.clone()]
    cuda = lambda ts: [_cuda(t) for t in ts]  # noqa: E731
    yield "cpu", _owner(), gts, anchors, levels
    yield "fp64_gt_fp32_anchors", _owner(), cuda([g.double() for g in gts]), cuda(anchors), levels
    yield "fp32_gt_fp64_anchors", _owner(), cuda(gts), cuda([x.double() for x in anchors]), levels
    yield "int_gt", _owner(), cuda([g.round().to(torch.int32) for g in gts]), cuda(anchors), levels
    yield "int_anchors", _owner(), cuda(gts), cuda([x.to(torch.int64) for x in anchors]), levels
    yield "mixed_gt_dtypes", _owner(), cuda([gts[0], gts[1].half()]), cuda(anchors), levels
    yield "mixed_anchor_dtypes", _owner(), cuda(gts), cuda([anchors[0], anchors[1].half()]), levels
    yield "one_gt_on_the_cpu", _owner(), [_cuda(gts[0]), gts[1]], cuda(anchors), levels
    yield "one_anchor_tensor_on_the_cpu", _owner(), cuda(gts), [_cuda(anchors[0]), anchors[1]], levels
    yield "fewer_targets_than_images", _owner(), cuda(gts[:1]), cuda(anchors), levels
    yield "more_targets_than_images", _owner(), cuda(gts), cuda(anchors[:1]), levels
    yield "empty_levels", _owner(), cuda(gts), cuda(anchors), []
    yield "tensor_radius", _owner(torch.tensor(1.5)), cuda(gts), cuda(anchors), levels


@pytest.mark.parametrize("label", [c[0] for c in _cases()])
def test_uncovered_inputs_take_the_reference_body(label, monkeypatch):
    _, owner, gts, anchors, levels = next(c for c in _cases() if c[0] == label)

    def run():
        try:
            return _call(owner, gts, anchors, levels)
        except Exception as e:          # the reference's own error (an empty level list) must be the one raised
            return type(e), str(e)

    expected = run()
    monkeypatch.setattr(det, "fcos_match_op", _refuse)
    vision_b200.install()
    try:
        got = run()
    finally:
        vision_b200.uninstall()
    if isinstance(expected, tuple) and isinstance(expected[0], type):
        assert got == expected
    else:
        _same(got, expected)


def test_tracing_takes_the_reference_body(monkeypatch):
    a, levels = _anchors()
    gts, anchors = [_cuda(_gt(3, 0))], [_cuda(a)]
    expected = _call(_owner(), gts, anchors, levels)
    monkeypatch.setattr(det, "fcos_match_op", _refuse)
    monkeypatch.setattr(tv, "_is_tracing", lambda: True)
    vision_b200.install()
    try:
        _same(_call(_owner(), gts, anchors, levels), expected)
    finally:
        vision_b200.uninstall()


def test_too_many_anchors_are_left_to_the_reference():
    gts = [_cuda(_gt(2, 0))]
    assert not det.fcos_match_supported(gts, [_cuda(torch.zeros(1, 4).expand(2**31, 4))], [2**31], 1.5)
    assert det.fcos_match_supported(gts, [_cuda(torch.zeros(1, 4).expand(2**31 - 1, 4))], [2**31 - 1], 1.5)


def test_covered_inputs_take_one_fused_call(monkeypatch):
    """The control for the cases above: the same stand-in inputs reach the op once for all images, with a background image,
    fp16 anchors against fp32 gt and the level list's first and last entries; head.compute_loss gets the op's result."""
    a, levels = _anchors()
    gts = [_cuda(_gt(3, 0)), _cuda(torch.zeros(0, 4)), _cuda(_gt(2, 1))]
    anchors = [_cuda(a.half()) for _ in range(3)]
    calls = []
    result = [torch.full((a.shape[0],), i) for i in range(3)]

    def fused(g, anc, radius, nlevels):
        calls.append((len(g), len(anc), radius, nlevels[0], nlevels[-1]))
        return result

    monkeypatch.setattr(det, "fcos_match_op", fused)
    vision_b200.install()
    try:
        got = _call(_owner(2.5), gts, anchors, levels)
    finally:
        vision_b200.uninstall()
    assert calls == [(3, 3, 2.5, levels[0], levels[-1])]
    assert got is result


def _bounds(n, first, last):
    lower, upper = ctypes.c_int64(), ctypes.c_int64()
    _lib.core().vb200_fcos_level_bounds(ctypes.c_int64(n), ctypes.c_int64(first), ctypes.c_int64(last), ctypes.byref(lower),
                                        ctypes.byref(upper))
    return lower.value, upper.value


@pytest.mark.parametrize("n", [0, 1, 7, 18134])
@pytest.mark.parametrize("first,last", [(3, 2), (0, 0), (5, 0), (10**6, 1), (3, 10**6), (-2, -3), (-10**6, -10**6), (7, 7)])
def test_level_bounds_follow_the_reference_slicing(n, first, last):
    """lower_bound[:first] = 0 and upper_bound[-last:] = inf as fcos.py:472-475 slices them; a last level of 0 anchors makes
    [-0:] the whole tensor and counts beyond N clamp."""
    lower = torch.ones(n)
    lower[:first] = 0
    upper = torch.ones(n)
    upper[-last:] = float("inf")
    lower_end, upper_begin = _bounds(n, first, last)
    assert torch.equal(lower == 0, torch.arange(n) < lower_end)
    assert torch.equal(upper == float("inf"), torch.arange(n) >= upper_begin)
    assert 0 <= lower_end <= n and 0 <= upper_begin <= n


def test_fake_op_gives_the_reference_shapes():
    from torch._subclasses.fake_tensor import FakeTensorMode

    _lib.load_ops()
    with FakeTensorMode():
        gts = [torch.empty(3, 4, device="cuda"), torch.empty(0, 4, device="cuda"), torch.empty(50, 4, device="cuda", dtype=torch.float16)]
        anchors = [torch.empty(n, 4, device="cuda", dtype=torch.float16) for n in (18134, 77, 0)]
        out = torch.ops.vision_b200.fcos_match(gts, anchors, 1.5, 14000, 20)
    assert [tuple(o.shape) for o in out] == [(18134,), (77,), (0,)]
    assert all(o.dtype == torch.int64 and o.device.type == "cuda" for o in out)
