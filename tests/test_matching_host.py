"""CPU suite: the training-target assignment of RegionProposalNetwork, RoIHeads and RetinaNet is rebound by install() and
restored by uninstall(); inputs the matching kernel does not cover keep running the reference body; the workspace query
answers without a GPU."""
import ctypes
import types

import pytest
import torch

tv = pytest.importorskip("torchvision")
from torchvision.models.detection import _utils as det_utils, retinanet, roi_heads, rpn  # noqa: E402
from torchvision.ops import boxes as box_ops  # noqa: E402

import vision_b200  # noqa: E402
from vision_b200 import detection as det  # noqa: E402

_METHODS = ((rpn.RegionProposalNetwork, "assign_targets_to_anchors"), (roi_heads.RoIHeads, "assign_targets_to_proposals"),
            (retinanet.RetinaNet, "compute_loss"))


class _SeenAsCuda(torch.Tensor):
    """A CPU tensor the coverage predicate takes for a CUDA one, so that each case below is refused for its own reason
    and the reference body can still run here."""

    @property
    def is_cuda(self):
        return True


def _boxes(n, seed, dtype=torch.float32):
    gen = torch.Generator().manual_seed(seed)
    xy = torch.rand(n, 2, generator=gen) * 200
    return torch.cat([xy, xy + torch.rand(n, 2, generator=gen) * 80 + 1], 1).to(dtype)


def _cuda(t):
    return t.as_subclass(_SeenAsCuda)


def _owners(matcher):
    """Stand-ins for the three modules: the methods read only these attributes."""
    head = types.SimpleNamespace(compute_loss=lambda targets, outputs, anchors, matched: matched)
    return (types.SimpleNamespace(box_similarity=box_ops.box_iou, proposal_matcher=matcher),
            types.SimpleNamespace(proposal_matcher=matcher),
            types.SimpleNamespace(proposal_matcher=matcher, head=head))


def _call_all(owners, gts, preds, labels):
    r, h, n = owners
    return (rpn.RegionProposalNetwork.assign_targets_to_anchors(r, preds, [{"boxes": g} for g in gts]),
            roi_heads.RoIHeads.assign_targets_to_proposals(h, preds, gts, labels),
            retinanet.RetinaNet.compute_loss(n, [{"boxes": g} for g in gts], {}, preds))


def _same(a, b):
    if isinstance(a, (list, tuple)):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            _same(x, y)
        return
    assert a.dtype == b.dtype and a.shape == b.shape and a.stride() == b.stride()
    assert torch.equal(torch.as_tensor(a), torch.as_tensor(b))


def test_install_rebinds_and_restores_the_three_methods():
    origs = [getattr(cls, name) for cls, name in _METHODS]
    vision_b200.install()
    try:
        for (cls, name), orig in zip(_METHODS, origs):
            assert getattr(cls, name) is not orig and getattr(cls, name).__wrapped__ is orig
    finally:
        vision_b200.uninstall()
    assert [getattr(cls, name) for cls, name in _METHODS] == origs


def _refuse(*a, **k):
    raise AssertionError("the fused path must not be taken for these inputs")


class _SubMatcher(det_utils.Matcher):
    pass


def _cases():
    gts, preds = [_boxes(3, 0), _boxes(2, 1)], [_boxes(40, 2), _boxes(30, 3)]
    labels = [torch.tensor([1, 2, 3]), torch.tensor([4, 5])]
    m = det_utils.Matcher(0.7, 0.3, True)
    yield "cpu", m, gts, preds, labels
    cuda = lambda ts: [_cuda(t) for t in ts]  # noqa: E731
    yield "ssd_matcher", det_utils.SSDMatcher(0.5), cuda(gts), cuda(preds), cuda(labels)
    yield "matcher_subclass", _SubMatcher(0.7, 0.3, True), cuda(gts), cuda(preds), cuda(labels)
    yield "fp64_gt_fp32_predictions", m, cuda([g.double() for g in gts]), cuda(preds), cuda(labels)
    yield "fp32_gt_fp64_predictions", m, cuda(gts), cuda([p.double() for p in preds]), cuda(labels)
    yield "int_gt", m, cuda([g.round().to(torch.int32) for g in gts]), cuda(preds), cuda(labels)
    yield "mixed_gt_dtypes", m, cuda([gts[0], gts[1].half()]), cuda(preds), cuda(labels)
    yield "one_side_cpu", m, [_cuda(gts[0]), gts[1]], cuda(preds), cuda(labels)
    yield "fewer_targets_than_images", m, cuda(gts[:1]), cuda(preds), cuda(labels[:1])


@pytest.mark.parametrize("label", [c[0] for c in _cases()])
def test_uncovered_inputs_take_the_reference_body(label, monkeypatch):
    _, matcher, gts, preds, labels = next(c for c in _cases() if c[0] == label)
    owners = _owners(matcher)
    expected = _call_all(owners, gts, preds, labels)
    monkeypatch.setattr(det, "match_boxes_op", _refuse)
    vision_b200.install()
    try:
        got = _call_all(owners, gts, preds, labels)
    finally:
        vision_b200.uninstall()
    _same(got, expected)


def test_other_similarity_and_tracing_take_the_reference_body(monkeypatch):
    gts, preds = [_cuda(_boxes(3, 0))], [_cuda(_boxes(40, 2))]
    r, _, _ = _owners(det_utils.Matcher(0.7, 0.3, True))
    r.box_similarity = lambda a, b: box_ops.box_iou(a, b)
    targets = [{"boxes": gts[0]}]
    expected = rpn.RegionProposalNetwork.assign_targets_to_anchors(r, preds, targets)
    monkeypatch.setattr(det, "match_boxes_op", _refuse)
    vision_b200.install()
    try:
        _same(rpn.RegionProposalNetwork.assign_targets_to_anchors(r, preds, targets), expected)
        r.box_similarity = box_ops.box_iou
        monkeypatch.setattr(tv, "_is_tracing", lambda: True)
        _same(rpn.RegionProposalNetwork.assign_targets_to_anchors(r, preds, targets), expected)
    finally:
        vision_b200.uninstall()


def test_too_many_predictions_are_left_to_the_reference():
    m = det_utils.Matcher(0.7, 0.3, True)
    huge = _cuda(torch.zeros(1, 4).expand(2**31, 4))
    assert not det.match_supported(m, [_cuda(_boxes(2, 0))], [huge])
    assert det.match_supported(m, [_cuda(_boxes(2, 0))], [_cuda(torch.zeros(1, 4).expand(2**31 - 1, 4))])


def test_covered_inputs_take_one_fused_call(monkeypatch):
    """The control for the cases above: the same stand-in inputs reach the op, once for all images, with the mode of each
    caller, including a background image and fp16 predictions against fp32 gt."""
    gts = [_cuda(_boxes(3, 0)), _cuda(torch.zeros(0, 4)), _cuda(_boxes(2, 1))]
    preds = [_cuda(_boxes(40, 2).half()), _cuda(_boxes(30, 3).half()), _cuda(_boxes(20, 4).half())]
    labels = [_cuda(torch.tensor([1, 2, 3])), _cuda(torch.zeros(0, dtype=torch.int64)), _cuda(torch.tensor([4, 5]))]
    calls = []

    def fused(g, p, lb, matcher, mode):
        calls.append((len(g), mode, lb is not None))
        return [torch.zeros(x.shape[0]) for x in p], [torch.zeros(x.shape[0]) for x in p]

    monkeypatch.setattr(det, "match_boxes_op", fused)
    vision_b200.install()
    try:
        _call_all(_owners(det_utils.Matcher(0.7, 0.3, True)), gts, preds, labels)
    finally:
        vision_b200.uninstall()
    assert calls == [(3, det.MATCH_RPN, False), (3, det.MATCH_ROI_HEADS, True), (3, det.MATCH_RAW, False)]


def test_no_predictions_raise_the_matcher_error_from_the_shapes():
    m = det_utils.Matcher(0.5, 0.5, False)
    with pytest.raises(ValueError, match="No proposal boxes available for one of the images during training"):
        det.match_boxes_op([_boxes(2, 0), torch.zeros(0, 4)], [_boxes(5, 1)[:0], _boxes(5, 2)], None, m, det.MATCH_RAW)


def test_matching_workspace_query_needs_no_gpu():
    from vision_b200 import _lib

    q = _lib.core().vb200_match_boxes_workspace_bytes
    q.restype = ctypes.c_size_t
    assert q(ctypes.c_int64(0), 0, 1) == 0
    assert q(ctypes.c_int64(100), 0, 0) == 0                # no low-quality matches: no gt maxima to keep
    assert q(ctypes.c_int64(100), 0, 1) == 512             # one 4-byte key per gt box, 256-byte aligned
    assert q(ctypes.c_int64(100), 3, 1) == 1024            # fp64: 8-byte keys
