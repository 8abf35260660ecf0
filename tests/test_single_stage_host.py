"""CPU suite: the single-stage detectors' postprocess_detections (RetinaNet, FCOS, SSD / SSDLite) are rebound by install()
and restored by uninstall(); inputs the fused kernel does not cover keep running the reference body; the workspace query
answers without a GPU."""
import ctypes

import pytest
import torch

tv = pytest.importorskip("torchvision")
from torchvision.models.detection import _utils as det_utils  # noqa: E402
from torchvision.models.detection.fcos import FCOS  # noqa: E402
from torchvision.models.detection.retinanet import RetinaNet  # noqa: E402
from torchvision.models.detection.ssd import SSD  # noqa: E402

import vision_b200  # noqa: E402
from vision_b200 import detection as det  # noqa: E402


def _bare(cls, coder, **attrs):
    """The model attributes postprocess_detections reads, without building a backbone."""
    m = cls.__new__(cls)
    m.box_coder = coder
    m.score_thresh, m.topk_candidates, m.nms_thresh, m.detections_per_img = 0.05, 1000, 0.5, 300
    for k, v in attrs.items():
        setattr(m, k, v)
    return m


def _anchors(n, gen, dtype):
    xy = torch.rand(n, 2, generator=gen) * 200
    wh = torch.rand(n, 2, generator=gen) * 60 + 4
    return torch.cat([xy, xy + wh], 1).to(dtype)


def _dense_inputs(num_images=2, levels=(48, 12), C=5, dtype=torch.float32, ctrness=False, seed=0):
    gen = torch.Generator().manual_seed(seed)
    total = sum(levels)
    cls = (torch.randn(num_images, total, C, generator=gen) * 2 - 2).to(dtype)
    reg = (torch.randn(num_images, total, 4, generator=gen) * 0.3).to(dtype)
    head = {"cls_logits": list(cls.split(levels, 1)), "bbox_regression": list(reg.split(levels, 1))}
    if ctrness:
        head["bbox_ctrness"] = list(torch.randn(num_images, total, 1, generator=gen).to(dtype).split(levels, 1))
    anchors = [list(_anchors(total, gen, dtype).split(levels)) for _ in range(num_images)]
    return head, anchors, [(180, 220), (200, 160)][:num_images]


def _ssd_inputs(num_images=2, A=64, C=6, dtype=torch.float32, seed=0):
    gen = torch.Generator().manual_seed(seed)
    head = {"cls_logits": torch.randn(num_images, A, C, generator=gen).to(dtype),
            "bbox_regression": (torch.randn(num_images, A, 4, generator=gen) * 0.3).to(dtype)}
    return head, [_anchors(A, gen, dtype) for _ in range(num_images)], [(180, 220), (200, 160)][:num_images]


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x.keys() == y.keys()
        for k in x:
            assert x[k].dtype == y[k].dtype and torch.equal(x[k], y[k]), k


def test_install_rebinds_and_restores_single_stage_postprocess():
    originals = {cls: cls.postprocess_detections for cls in (RetinaNet, FCOS, SSD)}
    vision_b200.install()
    try:
        for cls, orig in originals.items():
            assert cls.postprocess_detections is not orig
            assert cls.postprocess_detections.__wrapped__ is orig
    finally:
        vision_b200.uninstall()
    for cls, orig in originals.items():
        assert cls.postprocess_detections is orig


class _MyCoder(det_utils.BoxCoder):
    pass


def _cases():
    # (label, model, inputs): every one of these must take the reference body
    retina = _bare(RetinaNet, det_utils.BoxCoder(weights=(1.0, 1.0, 1.0, 1.0)))
    fcos = _bare(FCOS, det_utils.BoxLinearCoder(normalize_by_size=True), score_thresh=0.2)
    ssd = _bare(SSD, det_utils.BoxCoder(weights=(10.0, 10.0, 5.0, 5.0)), score_thresh=0.01, topk_candidates=400)
    yield "retinanet_cpu", retina, _dense_inputs()
    yield "fcos_cpu", fcos, _dense_inputs(ctrness=True)
    yield "ssd_cpu", ssd, _ssd_inputs()
    # fp16 heads: nothing passes a threshold of 1.0, so the reference's CPU body (no fp16 nms on CPU) completes
    yield "retinanet_fp16", _bare(RetinaNet, det_utils.BoxCoder(weights=(1.0, 1.0, 1.0, 1.0)), score_thresh=1.0), \
        _dense_inputs(dtype=torch.float16)
    yield "ssd_fp16", _bare(SSD, det_utils.BoxCoder(weights=(10.0, 10.0, 5.0, 5.0)), score_thresh=1.0), _ssd_inputs(dtype=torch.float16)
    yield "retinanet_subclassed_coder", _bare(RetinaNet, _MyCoder(weights=(1.0, 1.0, 1.0, 1.0))), _dense_inputs()
    yield "ssd_subclassed_coder", _bare(SSD, _MyCoder(weights=(10.0, 10.0, 5.0, 5.0)), score_thresh=0.01), _ssd_inputs()
    yield "fcos_unnormalized", _bare(FCOS, det_utils.BoxLinearCoder(normalize_by_size=False), score_thresh=0.2), _dense_inputs(ctrness=True)
    yield "retinanet_topk_above_capacity", _bare(RetinaNet, det_utils.BoxCoder(weights=(1.0, 1.0, 1.0, 1.0)),
                                                 topk_candidates=det.SINGLE_STAGE_MAX_TOPK + 1), _dense_inputs()


@pytest.mark.parametrize("label", [c[0] for c in _cases()])
def test_uncovered_inputs_take_the_reference_body(label, monkeypatch):
    _, model, (head, anchors, shapes) = next(c for c in _cases() if c[0] == label)
    expected = type(model).postprocess_detections(model, head, anchors, shapes)

    def refuse(*a, **k):
        raise AssertionError("the fused path must not be taken for these inputs")

    monkeypatch.setattr(det, "single_stage_postprocess", refuse)
    vision_b200.install()
    try:
        got = type(model).postprocess_detections(model, head, anchors, shapes)
    finally:
        vision_b200.uninstall()
    _same(got, expected)


def test_single_stage_workspace_query_needs_no_gpu():
    from vision_b200 import _lib

    lib = _lib.core()
    q = lib.vb200_single_stage_postprocess_workspace_bytes
    q.restype = ctypes.c_size_t
    retina = (ctypes.c_int64 * 5)(122400, 30600, 7650, 2016, 567)
    one = q(0, 1, 5, retina, 91, ctypes.c_int64(1000), ctypes.c_int64(300))
    eight = q(0, 8, 5, retina, 91, ctypes.c_int64(1000), ctypes.c_int64(300))
    assert one > 0 and eight > one
    # sized from shapes and k: about 5 levels x (hist + pairs) + candidates + the batched_nms workspace, far below the logits
    assert one < 122400 * 91 * 4
    ssd = (ctypes.c_int64 * 1)(8732)
    assert q(2, 8, 1, ssd, 91, ctypes.c_int64(400), ctypes.c_int64(200)) > 0
    assert q(0, 1, 5, retina, 91, ctypes.c_int64(det.SINGLE_STAGE_MAX_TOPK + 1), ctypes.c_int64(300)) == 0
