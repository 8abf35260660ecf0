"""CPU suite: FCOSHead.compute_loss is rebound by install() and restored by uninstall(); inputs the fused FCOS loss kernels
do not cover keep running the reference body; covered inputs reach each op once; the fake ops give the shapes and dtypes
the real ones return."""
import pytest
import torch

tv = pytest.importorskip("torchvision")
from torchvision.models.detection import _utils as det_utils, fcos, retinanet  # noqa: E402

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


def _inputs(B=2, A=40, C=3, seed=0):
    gen = torch.Generator().manual_seed(seed)
    xy = torch.rand(A, 2, generator=gen) * 100
    anchors = torch.cat([xy, xy + torch.rand(A, 2, generator=gen) * 20 + 4], 1)
    targets, matched = [], []
    for _ in range(B):
        pick = torch.randint(0, A, (3,), generator=gen)
        targets.append({"boxes": anchors[pick] + 1, "labels": torch.randint(0, C, (3,), generator=gen)})
        matched.append(torch.randint(-1, 3, (A,), generator=gen))
    outputs = {"cls_logits": torch.randn(B, A, C, generator=gen), "bbox_regression": torch.randn(B, A, 4, generator=gen) * 0.1,
               "bbox_ctrness": torch.randn(B, A, 1, generator=gen)}
    return targets, outputs, [anchors] * B, matched


def _cuda_inputs(**kw):
    targets, outputs, anchors, matched = _inputs(**kw)
    targets = [{"boxes": _cuda(t["boxes"]), "labels": _cuda(t["labels"])} for t in targets]
    return targets, {k: _cuda(v) for k, v in outputs.items()}, [_cuda(a) for a in anchors], [_cuda(m) for m in matched]


def _head(coder=None):
    head = fcos.FCOSHead(32, 1, 3, num_convs=1)
    if coder is not None:
        head.box_coder = coder
    return head


def _refuse(*a, **k):
    raise AssertionError("the fused path must not be taken for these inputs")


def test_install_rebinds_and_restores_the_head_loss():
    orig = fcos.FCOSHead.compute_loss
    retina = {(retinanet.RetinaNetClassificationHead, "compute_loss"): retinanet.RetinaNetClassificationHead.compute_loss,
              (retinanet.RetinaNetRegressionHead, "compute_loss"): retinanet.RetinaNetRegressionHead.compute_loss}
    vision_b200.install()
    try:
        from vision_b200 import _install

        assert fcos.FCOSHead.compute_loss.__wrapped__ is orig
        assert _install._state["fcos_losses"] == {(fcos.FCOSHead, "compute_loss"): orig}
        assert _install._state["losses"] == retina
    finally:
        vision_b200.uninstall()
    assert fcos.FCOSHead.compute_loss is orig


class _OtherCoder(det_utils.BoxLinearCoder):
    pass


def _cases():
    targets, outputs, anchors, matched = _cuda_inputs()
    plain = _inputs()
    yield "cpu", _head(), *plain
    yield "fp16_logits", _head(), targets, {**outputs, "cls_logits": _cuda(outputs["cls_logits"].half())}, anchors, matched
    yield "bf16_regression", _head(), targets, {**outputs, "bbox_regression": _cuda(outputs["bbox_regression"].bfloat16())}, anchors, matched
    yield "coder_subclass", _head(_OtherCoder(True)), targets, outputs, anchors, matched
    yield "box_coder", _head(det_utils.BoxCoder((1.0, 1.0, 1.0, 1.0))), targets, outputs, anchors, matched
    yield "empty_targets", _head(), [], {k: v[:0] for k, v in outputs.items()}, [], []
    yield "fewer_matches_than_images", _head(), targets, outputs, anchors, matched[:1]
    yield "cls_logits_not_dense", _head(), targets, {**outputs, "cls_logits": _cuda(outputs["cls_logits"].transpose(1, 2).contiguous()
                                                                                   .transpose(1, 2))}, anchors, matched
    yield "ctrness_a_differs", _head(), targets, {**outputs, "bbox_ctrness": outputs["bbox_ctrness"][:, :-1]}, anchors, matched
    yield "fp64_anchors", _head(), targets, outputs, [_cuda(a.double()) for a in anchors], matched
    yield "int32_labels", _head(), [{"boxes": t["boxes"], "labels": _cuda(t["labels"].int())} for t in targets], outputs, anchors, matched
    yield "one_gt_on_the_cpu", _head(), [targets[0], plain[0][1]], outputs, anchors, matched


def _outcome(fn):
    try:
        return fn()
    except Exception as e:          # the reference's own error must be the one raised
        return type(e), str(e)


def _same(got, expected):
    if isinstance(expected, tuple) and isinstance(expected[0], type):
        assert got == expected
    else:
        assert got.keys() == expected.keys()
        for k in expected:
            # random matches put anchor centres outside their gt box, so a centre-ness target (and that loss) may be NaN
            torch.testing.assert_close(torch.as_tensor(got[k]), torch.as_tensor(expected[k]), rtol=0, atol=0, equal_nan=True)


def _run_refused(head, targets, outputs, anchors, matched, monkeypatch, tracing=False):
    run = lambda: fcos.FCOSHead.compute_loss(head, targets, outputs, anchors, matched)  # noqa: E731
    expected = _outcome(run)
    monkeypatch.setattr(det, "fcos_cls_loss_op", _refuse)
    monkeypatch.setattr(det, "fcos_box_loss_op", _refuse)
    if tracing:
        monkeypatch.setattr(tv, "_is_tracing", lambda: True)
    vision_b200.install()
    try:
        got = _outcome(run)
    finally:
        vision_b200.uninstall()
    _same(got, expected)


@pytest.mark.parametrize("label", [c[0] for c in _cases()])
def test_uncovered_inputs_take_the_reference_body(label, monkeypatch):
    _run_refused(*next(c for c in _cases() if c[0] == label)[1:], monkeypatch)


def test_tracing_takes_the_reference_body(monkeypatch):
    _run_refused(_head(), *_cuda_inputs(), monkeypatch, tracing=True)


@pytest.mark.parametrize("normalize", [True, False])
def test_covered_inputs_take_one_fused_call_each(normalize, monkeypatch):
    """The control for the cases above: the same stand-in inputs reach each op once for all images, and the head returns
    the reference's three keys with the ops' results."""
    targets, outputs, anchors, matched = _cuda_inputs()
    calls = []

    def cls_op(logits, m, labels):
        calls.append(("cls", logits, len(m), len(labels)))
        return torch.tensor(1.5)

    def box_op(regression, ctrness, a, boxes, labels, m, norm):
        calls.append(("box", regression, ctrness, len(a), len(boxes), len(labels), len(m), norm))
        return torch.tensor(2.5), torch.tensor(3.5)

    monkeypatch.setattr(det, "fcos_cls_loss_op", cls_op)
    monkeypatch.setattr(det, "fcos_box_loss_op", box_op)
    vision_b200.install()
    try:
        got = fcos.FCOSHead.compute_loss(_head(det_utils.BoxLinearCoder(normalize)), targets, outputs, anchors, matched)
    finally:
        vision_b200.uninstall()
    assert list(got) == ["classification", "bbox_regression", "bbox_ctrness"]
    assert [got[k].item() for k in got] == [1.5, 2.5, 3.5]
    assert sorted(c[0] for c in calls) == ["box", "cls"]
    cls_call, box_call = sorted(calls, key=lambda c: c[0] != "cls")
    assert cls_call[1] is outputs["cls_logits"] and cls_call[2:] == (2, 2)
    assert box_call[1] is outputs["bbox_regression"] and box_call[2] is outputs["bbox_ctrness"]
    assert box_call[3:] == (2, 2, 2, 2, normalize)


def test_fake_ops_give_the_real_shapes_and_dtypes():
    from torch._subclasses.fake_tensor import FakeTensorMode

    _lib.load_ops()
    ops = torch.ops.vision_b200
    with FakeTensorMode():
        logits = torch.empty(3, 1000, 91, device="cuda")
        regression = torch.empty(3, 1000, 4, device="cuda")
        ctrness = torch.empty(3, 1000, 1, device="cuda")
        matched = [torch.empty(1000, dtype=torch.int64, device="cuda") for _ in range(3)]
        labels = [torch.empty(n, dtype=torch.int64, device="cuda") for n in (3, 0, 50)]
        boxes = [torch.empty(n, 4, device="cuda") for n in (3, 0, 50)]
        anchors = [torch.empty(1000, 4, device="cuda") for _ in range(3)]
        g = torch.empty((), device="cuda")
        loss, count = ops.fcos_cls_loss(logits, matched, labels)
        grad = ops.fcos_cls_loss_backward(g, logits, matched, labels, count)
        lbox, lctr, bcount = ops.fcos_box_loss(regression, ctrness, anchors, boxes, labels, matched, True)
        gbox, gctr = ops.fcos_box_loss_backward(g, None, regression, ctrness, anchors, boxes, labels, matched, True, bcount)
    for l in (loss, lbox, lctr):
        assert l.shape == () and l.dtype == torch.float32 and l.device.type == "cuda"
    for c in (count, bcount):
        assert c.shape == () and c.dtype == torch.int64 and c.device.type == "cuda"
    assert tuple(grad.shape) == (3, 1000, 91) and grad.dtype == torch.float32 and grad.is_contiguous()
    assert tuple(gbox.shape) == (3, 1000, 4) and gbox.dtype == torch.float32 and gbox.is_contiguous()
    assert tuple(gctr.shape) == (3, 1000, 1) and gctr.dtype == torch.float32 and gctr.is_contiguous()
