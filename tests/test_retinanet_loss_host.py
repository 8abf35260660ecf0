"""CPU suite: RetinaNet's two head-loss methods are rebound by install() and restored by uninstall(); inputs the fused loss
kernels do not cover keep running the reference body, each head on its own; the fake ops give the shapes and dtypes the
real ones return."""
import types

import pytest
import torch

tv = pytest.importorskip("torchvision")
from torchvision.models.detection import _utils as det_utils, retinanet  # noqa: E402

import vision_b200  # noqa: E402
from vision_b200 import _lib, detection as det  # noqa: E402


class _SeenAsCuda(torch.Tensor):
    """A CPU tensor the coverage predicates take for a CUDA one, so that each case below is refused for its own reason and
    the reference body can still run here."""

    @property
    def is_cuda(self):
        return True


def _cuda(t):
    return t.as_subclass(_SeenAsCuda)


def _inputs(B=2, A=40, C=3, seed=0):
    gen = torch.Generator().manual_seed(seed)
    xy = torch.rand(A, 2, generator=gen) * 100
    anchors = torch.cat([xy, xy + torch.rand(A, 2, generator=gen) * 20 + 4], 1)
    targets, matched = [], []
    for i in range(B):
        pick = torch.randint(0, A, (3,), generator=gen)
        targets.append({"boxes": anchors[pick] + 1, "labels": torch.randint(0, C, (3,), generator=gen)})
        matched.append(torch.randint(-2, 3, (A,), generator=gen))
    logits = torch.randn(B, A, C, generator=gen)
    regression = torch.randn(B, A, 4, generator=gen)
    return targets, matched, logits, regression, [anchors] * B


def _cuda_inputs(**kw):
    targets, matched, logits, regression, anchors = _inputs(**kw)
    targets = [{"boxes": _cuda(t["boxes"]), "labels": _cuda(t["labels"])} for t in targets]
    return targets, [_cuda(m) for m in matched], _cuda(logits), _cuda(regression), [_cuda(a) for a in anchors]


def _head(cls_head, box_head):
    """A stand-in RetinaNetHead: its compute_loss reads only the two heads."""
    return types.SimpleNamespace(classification_head=cls_head, regression_head=box_head)


def _refuse(*a, **k):
    raise AssertionError("the fused path must not be taken for these inputs")


def test_install_rebinds_and_restores_both_head_losses():
    cls_orig = retinanet.RetinaNetClassificationHead.compute_loss
    box_orig = retinanet.RetinaNetRegressionHead.compute_loss
    head_orig = retinanet.RetinaNetHead.compute_loss
    vision_b200.install()
    try:
        from vision_b200 import _install

        assert retinanet.RetinaNetClassificationHead.compute_loss.__wrapped__ is cls_orig
        assert retinanet.RetinaNetRegressionHead.compute_loss.__wrapped__ is box_orig
        assert retinanet.RetinaNetHead.compute_loss is head_orig
        assert _install._state["losses"] == {(retinanet.RetinaNetClassificationHead, "compute_loss"): cls_orig,
                                             (retinanet.RetinaNetRegressionHead, "compute_loss"): box_orig}
    finally:
        vision_b200.uninstall()
    assert retinanet.RetinaNetClassificationHead.compute_loss is cls_orig
    assert retinanet.RetinaNetRegressionHead.compute_loss is box_orig


def _cls_cases():
    targets, matched, logits, _, _ = _cuda_inputs()
    plain_t, plain_m, plain_l, _, _ = _inputs()
    head = retinanet.RetinaNetClassificationHead(4, 1, 3)
    yield "cpu", head, plain_t, plain_m, plain_l
    yield "empty_targets", head, [], [], logits[:0]
    yield "fewer_matches_than_targets", head, targets, matched[:1], logits
    yield "batch_of_logits_differs", head, targets[:1], matched[:1], logits
    yield "fp16_logits", head, targets, matched, _cuda(logits.half())
    yield "bf16_logits", head, targets, matched, _cuda(logits.bfloat16())
    yield "fp64_logits", head, targets, matched, _cuda(logits.double())
    yield "classes_not_unit_stride", head, targets, matched, _cuda(logits.transpose(1, 2).contiguous().transpose(1, 2))
    yield "not_three_dimensional", head, targets, matched, _cuda(logits.reshape(-1, 3))
    yield "int32_matches", head, targets, [_cuda(m.int()) for m in matched], logits
    yield "matches_not_one_dimensional", head, targets, [_cuda(m[:, None]) for m in matched], logits
    yield "int32_labels", head, [{"boxes": t["boxes"], "labels": _cuda(t["labels"].int())} for t in targets], matched, logits
    yield "one_match_on_the_cpu", head, targets, [matched[0], plain_m[1]], logits
    yield "one_label_on_the_cpu", head, [targets[0], plain_t[1]], matched, logits
    odd = retinanet.RetinaNetClassificationHead(4, 1, 3)
    odd.BETWEEN_THRESHOLDS = -3
    yield "other_between_thresholds_code", odd, targets, matched, logits


def _box_cases():
    targets, matched, _, regression, anchors = _cuda_inputs()
    plain_t, plain_m, _, plain_r, plain_a = _inputs()

    def head(loss_type="l1", coder=None):
        h = retinanet.RetinaNetRegressionHead(4, 1)
        h._loss_type = loss_type
        if coder is not None:
            h.box_coder = coder
        return h

    class Coder(det_utils.BoxCoder):
        pass

    yield "cpu", head(), plain_t, plain_m, plain_r, plain_a
    yield "empty_targets", head(), [], [], regression[:0], []
    yield "giou", head("giou"), targets, matched, regression, anchors
    yield "smooth_l1", head("smooth_l1"), targets, matched, regression, anchors
    yield "box_coder_subclass", head(coder=Coder((1.0, 1.0, 1.0, 1.0))), targets, matched, regression, anchors
    yield "fp64_anchors", head(), targets, matched, regression, [_cuda(a.double()) for a in anchors]
    yield "fp64_gt_boxes", head(), [{"boxes": _cuda(t["boxes"].double()), "labels": t["labels"]} for t in targets], matched, regression, anchors
    yield "fp16_regression", head(), targets, matched, _cuda(regression.half()), anchors
    yield "fewer_anchor_tensors_than_targets", head(), targets, matched, regression, anchors[:1]
    yield "int32_matches", head(), targets, [_cuda(m.int()) for m in matched], regression, anchors
    yield "one_anchor_tensor_on_the_cpu", head(), targets, matched, regression, [anchors[0], plain_a[1]]
    yield "one_gt_on_the_cpu", head(), [targets[0], plain_t[1]], matched, regression, anchors


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


@pytest.mark.parametrize("label", [c[0] for c in _cls_cases()])
def test_uncovered_classification_inputs_take_the_reference_body(label, monkeypatch):
    _, head, targets, matched, logits = next(c for c in _cls_cases() if c[0] == label)
    run = lambda: retinanet.RetinaNetClassificationHead.compute_loss(head, targets, {"cls_logits": logits}, matched)  # noqa: E731
    expected = _outcome(run)
    monkeypatch.setattr(det, "retinanet_cls_loss_op", _refuse)
    vision_b200.install()
    try:
        got = _outcome(run)
    finally:
        vision_b200.uninstall()
    _same(got, expected)


@pytest.mark.parametrize("label", [c[0] for c in _box_cases()])
def test_uncovered_regression_inputs_take_the_reference_body(label, monkeypatch):
    _, head, targets, matched, regression, anchors = next(c for c in _box_cases() if c[0] == label)
    run = lambda: retinanet.RetinaNetRegressionHead.compute_loss(head, targets, {"bbox_regression": regression}, anchors, matched)  # noqa: E731
    expected = _outcome(run)
    monkeypatch.setattr(det, "retinanet_box_loss_op", _refuse)
    vision_b200.install()
    try:
        got = _outcome(run)
    finally:
        vision_b200.uninstall()
    _same(got, expected)


def test_tracing_takes_the_reference_body(monkeypatch):
    targets, matched, logits, regression, anchors = _cuda_inputs()
    cls_head, box_head = retinanet.RetinaNetClassificationHead(4, 1, 3), retinanet.RetinaNetRegressionHead(4, 1)
    outputs = {"cls_logits": logits, "bbox_regression": regression}
    expected = retinanet.RetinaNetHead.compute_loss(_head(cls_head, box_head), targets, outputs, anchors, matched)
    monkeypatch.setattr(det, "retinanet_cls_loss_op", _refuse)
    monkeypatch.setattr(det, "retinanet_box_loss_op", _refuse)
    monkeypatch.setattr(tv, "_is_tracing", lambda: True)
    vision_b200.install()
    try:
        got = retinanet.RetinaNetHead.compute_loss(_head(cls_head, box_head), targets, outputs, anchors, matched)
    finally:
        vision_b200.uninstall()
    for k in expected:
        assert torch.equal(got[k], expected[k])


def test_too_many_logits_are_left_to_the_reference():
    """A * C of 2^31 or more goes to the reference (the kernels index an image with 32 bits); just below is fused."""
    head = retinanet.RetinaNetClassificationHead(4, 1, 2)

    def case(A):
        logits = _cuda(torch.empty(1, A, 2, device="meta"))
        matched = [_cuda(torch.empty(A, dtype=torch.int64, device="meta"))]
        targets = [{"labels": _cuda(torch.empty(3, dtype=torch.int64, device="meta"))}]
        return det.retinanet_cls_loss_supported(head, targets, logits, matched)

    assert not case(2**30)
    assert case(2**30 - 1)


def test_covered_inputs_take_one_fused_call_each(monkeypatch):
    """The control for the cases above: the same stand-in inputs reach each op once for all images, with the logits, the
    labels, the boxes and the coder's weights as fp32 rounds them; RetinaNetHead.compute_loss returns the ops' results."""
    targets, matched, logits, regression, anchors = _cuda_inputs()
    calls = []

    def cls_op(lg, m, labels):
        calls.append(("cls", lg, len(m), [l.dtype for l in labels]))
        return torch.tensor(1.5)

    def box_op(r, a, boxes, m, weights):
        calls.append(("box", r, len(a), len(boxes), len(m), weights))
        return torch.tensor(2.5)

    monkeypatch.setattr(det, "retinanet_cls_loss_op", cls_op)
    monkeypatch.setattr(det, "retinanet_box_loss_op", box_op)
    box_head = retinanet.RetinaNetRegressionHead(4, 1)
    box_head.box_coder = det_utils.BoxCoder((10.0, 10.0, 5.0, 0.1))
    outputs = {"cls_logits": logits, "bbox_regression": regression}
    vision_b200.install()
    try:
        got = retinanet.RetinaNetHead.compute_loss(_head(retinanet.RetinaNetClassificationHead(4, 1, 3), box_head), targets,
                                                   outputs, anchors, matched)
    finally:
        vision_b200.uninstall()
    assert got["classification"].item() == 1.5 and got["bbox_regression"].item() == 2.5
    assert [c[0] for c in calls] == ["cls", "box"]
    assert calls[0][1] is logits and calls[0][2:] == (2, [torch.int64, torch.int64])
    assert calls[1][1] is regression and calls[1][2:5] == (2, 2, 2)
    assert calls[1][5] == [10.0, 10.0, 5.0, float(torch.tensor(0.1, dtype=torch.float32))]


def test_v2_keeps_its_giou_regression_while_classification_is_fused(monkeypatch):
    """retinanet_resnet50_fpn_v2 regresses boxes with GIoU: its regression head falls back to the reference on its own while
    its classification head takes the fused op."""
    from torchvision.models.detection import retinanet_resnet50_fpn_v2

    model = retinanet_resnet50_fpn_v2(weights=None, weights_backbone=None, num_classes=3)
    assert model.head.regression_head._loss_type == "giou"
    targets, matched, logits, regression, anchors = _cuda_inputs()
    outputs = {"cls_logits": logits, "bbox_regression": regression}
    expected = model.head.compute_loss(targets, outputs, anchors, matched)
    monkeypatch.setattr(det, "retinanet_cls_loss_op", lambda *a: torch.tensor(7.0))
    monkeypatch.setattr(det, "retinanet_box_loss_op", _refuse)
    vision_b200.install()
    try:
        got = model.head.compute_loss(targets, outputs, anchors, matched)
    finally:
        vision_b200.uninstall()
    assert got["classification"].item() == 7.0
    assert torch.equal(got["bbox_regression"], expected["bbox_regression"])


def test_fake_ops_give_the_real_shapes_and_dtypes():
    from torch._subclasses.fake_tensor import FakeTensorMode

    _lib.load_ops()
    ops = torch.ops.vision_b200
    with FakeTensorMode():
        logits = torch.empty(3, 1000, 91, device="cuda")
        regression = torch.empty(3, 1000, 4, device="cuda")
        matched = [torch.empty(1000, dtype=torch.int64, device="cuda") for _ in range(3)]
        labels = [torch.empty(n, dtype=torch.int64, device="cuda") for n in (3, 0, 50)]
        boxes = [torch.empty(n, 4, device="cuda") for n in (3, 0, 50)]
        anchors = [torch.empty(1000, 4, device="cuda") for _ in range(3)]
        loss, counts = ops.retinanet_cls_loss(logits, matched, labels)
        grad = ops.retinanet_cls_loss_backward(torch.empty((), device="cuda"), logits, matched, labels, counts)
        bloss, bcounts = ops.retinanet_box_loss(regression, anchors, boxes, matched, [1.0, 1.0, 1.0, 1.0])
        bgrad = ops.retinanet_box_loss_backward(torch.empty((), device="cuda"), regression, anchors, boxes, matched, [1.0] * 4, bcounts)
    for l, c in ((loss, counts), (bloss, bcounts)):
        assert l.shape == () and l.dtype == torch.float32 and l.device.type == "cuda"
        assert tuple(c.shape) == (3,) and c.dtype == torch.int64 and c.device.type == "cuda"
    assert tuple(grad.shape) == (3, 1000, 91) and grad.dtype == torch.float32 and grad.is_contiguous()
    assert tuple(bgrad.shape) == (3, 1000, 4) and bgrad.dtype == torch.float32 and bgrad.is_contiguous()
