"""CPU suite: roi_heads.maskrcnn_loss is rebound by install() and restored by uninstall(); inputs the fused mask-loss kernels
do not cover keep running the reference body; the fake ops give the shapes and dtypes the real ones return."""
import pytest
import torch

tv = pytest.importorskip("torchvision")
from torchvision.models.detection import roi_heads  # noqa: E402

import vision_b200  # noqa: E402
from vision_b200 import _lib, detection as det  # noqa: E402


class _SeenAsCuda(torch.Tensor):
    """A CPU tensor the coverage predicate takes for a CUDA one, so that each case below is refused for its own reason and
    the reference body can still run here."""

    @property
    def is_cuda(self):
        return True


def _cuda(t):
    return t.as_subclass(_SeenAsCuda)


def _inputs(P=(3, 2), G=(2, 4), C=5, M=7, H=20, W=24, seed=0):
    gen = torch.Generator().manual_seed(seed)
    proposals, masks, labels, matched = [], [], [], []
    for p, g in zip(P, G):
        xy = torch.rand(p, 2, generator=gen) * 10
        proposals.append(torch.cat([xy, xy + 2 + torch.rand(p, 2, generator=gen) * 10], 1))
        masks.append(torch.rand(g, H, W, generator=gen) > 0.5)
        labels.append(torch.randint(1, C, (g,), generator=gen))
        matched.append(torch.randint(0, g, (p,), generator=gen))
    masks = [m.to(torch.uint8) for m in masks]
    logits = torch.randn(sum(P), C, M, M, generator=gen)
    return logits, proposals, masks, labels, matched


def _cuda_inputs(**kw):
    logits, proposals, masks, labels, matched = _inputs(**kw)
    return _cuda(logits), [_cuda(p) for p in proposals], [_cuda(m) for m in masks], [_cuda(l) for l in labels], [_cuda(m) for m in matched]


def _refuse(*a, **k):
    raise AssertionError("the fused path must not be taken for these inputs")


def test_install_rebinds_and_restores_maskrcnn_loss():
    orig = roi_heads.maskrcnn_loss
    vision_b200.install()
    try:
        from vision_b200 import _install

        assert roi_heads.maskrcnn_loss is not orig and roi_heads.maskrcnn_loss.__wrapped__ is orig
        assert _install._state["orig_mask_loss"] is orig
        assert (roi_heads.RoIHeads, "maskrcnn_loss") not in _install._state["losses"]
    finally:
        vision_b200.uninstall()
    assert roi_heads.maskrcnn_loss is orig


def _cases():
    logits, proposals, masks, labels, matched = _cuda_inputs()
    plain = _inputs()
    yield "cpu", plain
    yield "one_mask_stack_on_the_cpu", (logits, proposals, [masks[0], plain[2][1]], labels, matched)
    yield "one_proposal_tensor_on_the_cpu", (logits, [proposals[0], plain[1][1]], masks, labels, matched)
    yield "fp16_logits", (_cuda(logits.half()), proposals, masks, labels, matched)
    yield "bf16_logits", (_cuda(logits.bfloat16()), proposals, masks, labels, matched)
    yield "fp64_logits", (_cuda(logits.double()), proposals, masks, labels, matched)
    yield "logits_not_dense", (_cuda(logits.transpose(2, 3)), proposals, masks, labels, matched)
    yield "logits_not_square", (_cuda(logits[:, :, :, :6].contiguous()), proposals, masks, labels, matched)
    yield "logits_not_four_dimensional", (_cuda(logits.reshape(5, 5, -1)), proposals, masks, labels, matched)
    yield "rows_differ_from_proposals", (_cuda(logits[:4].contiguous()), proposals, masks, labels, matched)
    yield "fp32_masks", (logits, proposals, [_cuda(m.float()) for m in masks], labels, matched)
    yield "masks_not_three_dimensional", (logits, proposals, [_cuda(m[0]) for m in masks], labels, matched)
    yield "fp64_proposals", (logits, [_cuda(p.double()) for p in proposals], masks, labels, matched)
    yield "proposals_not_four_wide", (logits, [_cuda(torch.cat([p, p[:, :1]], 1)) for p in proposals], masks, labels, matched)
    yield "int32_matches", (logits, proposals, masks, labels, [_cuda(m.int()) for m in matched])
    yield "matches_not_one_dimensional", (logits, proposals, masks, labels, [_cuda(m[:, None]) for m in matched])
    yield "int32_labels", (logits, proposals, masks, [_cuda(l.int()) for l in labels], matched)
    yield "fewer_mask_stacks_than_images", (logits, proposals, masks[:1], labels, matched)
    empty = _cuda_inputs(P=(0, 0))
    yield "no_positives", empty


def _outcome(fn):
    try:
        return fn()
    except Exception as e:          # the reference's own error must be the one raised
        return type(e), str(e)


def _same(got, expected):
    if isinstance(expected, tuple) and isinstance(expected[0], type):
        assert got == expected
    else:
        assert torch.equal(torch.as_tensor(got), torch.as_tensor(expected))


@pytest.mark.parametrize("label", [c[0] for c in _cases()])
def test_uncovered_inputs_take_the_reference_body(label, monkeypatch):
    args = next(c for c in _cases() if c[0] == label)[1]
    run = lambda: roi_heads.maskrcnn_loss(*args)  # noqa: E731
    expected = _outcome(run)
    monkeypatch.setattr(det, "maskrcnn_loss_op", _refuse)
    vision_b200.install()
    try:
        got = _outcome(run)
    finally:
        vision_b200.uninstall()
    _same(got, expected)


def test_tracing_takes_the_reference_body(monkeypatch):
    args = _cuda_inputs()
    expected = roi_heads.maskrcnn_loss(*args)
    monkeypatch.setattr(det, "maskrcnn_loss_op", _refuse)
    monkeypatch.setattr(tv, "_is_tracing", lambda: True)
    vision_b200.install()
    try:
        got = roi_heads.maskrcnn_loss(*args)
    finally:
        vision_b200.uninstall()
    assert torch.equal(got, expected)


def test_too_many_logits_are_left_to_the_reference():
    """P * C * M * M of 2^31 or more goes to the reference (the kernels index the logits with 32 bits); just below is fused."""

    def case(P):
        logits = _cuda(torch.empty(P, 2, 32, 32, device="meta"))
        proposals = [_cuda(torch.empty(P, 4, device="meta"))]
        masks = [_cuda(torch.empty(3, 64, 64, dtype=torch.uint8, device="meta"))]
        labels = [_cuda(torch.empty(3, dtype=torch.int64, device="meta"))]
        matched = [_cuda(torch.empty(P, dtype=torch.int64, device="meta"))]
        return det.maskrcnn_loss_supported(logits, proposals, masks, labels, matched)

    assert not case(2**20)
    assert case(2**20 - 1)


def test_covered_inputs_take_one_fused_call(monkeypatch):
    """The control for the cases above: the same stand-in inputs reach the op once for all images, bool masks included, and
    the rebound maskrcnn_loss returns the op's loss."""
    logits, proposals, masks, labels, matched = _cuda_inputs()
    masks = [masks[0], _cuda(masks[1].bool())]
    calls = []

    def op(lg, p, g, l, m):
        calls.append((lg, len(p), [t.dtype for t in g], len(l), len(m)))
        return torch.tensor(0.75), None

    monkeypatch.setattr(det, "maskrcnn_loss_op", op)
    vision_b200.install()
    try:
        got = roi_heads.maskrcnn_loss(logits, proposals, masks, labels, matched)
    finally:
        vision_b200.uninstall()
    assert got.item() == 0.75
    assert len(calls) == 1 and calls[0][0] is logits and calls[0][1:] == (2, [torch.uint8, torch.bool], 2, 2)


def test_fake_ops_give_the_real_shapes_and_dtypes():
    from torch._subclasses.fake_tensor import FakeTensorMode

    _lib.load_ops()
    ops = torch.ops.vision_b200
    with FakeTensorMode():
        logits = torch.empty(256, 91, 28, 28, device="cuda")
        proposals = [torch.empty(128, 4, device="cuda") for _ in range(2)]
        masks = [torch.empty(n, 800, 1088, dtype=torch.uint8, device="cuda") for n in (7, 50)]
        labels = [torch.empty(n, dtype=torch.int64, device="cuda") for n in (7, 50)]
        matched = [torch.empty(128, dtype=torch.int64, device="cuda") for _ in range(2)]
        loss, targets = ops.maskrcnn_loss(logits, proposals, masks, labels, matched)
        grad = ops.maskrcnn_loss_backward(torch.empty((), device="cuda"), logits, targets, labels, matched)
    assert loss.shape == () and loss.dtype == torch.float32 and loss.device.type == "cuda"
    assert tuple(targets.shape) == (256, 28, 28) and targets.dtype == torch.float32
    assert tuple(grad.shape) == (256, 91, 28, 28) and grad.dtype == torch.float32 and grad.is_contiguous()
