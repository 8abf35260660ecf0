"""CPU suite: Keypoint R-CNN's keypointrcnn_inference / heatmaps_to_keypoints are rebound by install() and restored by
uninstall(); inputs the keypoint kernel does not cover keep running the reference body; the workspace query answers without
a GPU."""
import ctypes

import pytest
import torch

tv = pytest.importorskip("torchvision")
from torchvision.models.detection import roi_heads  # noqa: E402

import vision_b200  # noqa: E402
from vision_b200 import detection as det  # noqa: E402


class _SeenAsCuda(torch.Tensor):
    """A CPU tensor the coverage predicate takes for a CUDA one, so that each case below is refused for its own reason
    and the reference body can still run here."""

    @property
    def is_cuda(self):
        return True


def _inputs(K=3, N=4, H=8, W=8, maps_dtype=torch.float32, rois_dtype=torch.float32, seed=0):
    gen = torch.Generator().manual_seed(seed)
    maps = torch.randn(K, N, H, W, generator=gen).to(maps_dtype)
    xy = torch.rand(K, 2, generator=gen) * 50
    rois = torch.cat([xy, xy + torch.rand(K, 2, generator=gen) * 30 + 2], 1).to(rois_dtype)
    return maps, rois


def _seen_as_cuda(maps, rois):
    return maps.as_subclass(_SeenAsCuda), rois.as_subclass(_SeenAsCuda)


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        if isinstance(x, (list, tuple)):
            _same(x, y)
            continue
        assert x.dtype == y.dtype and x.shape == y.shape and x.stride() == y.stride()
        assert torch.equal(torch.as_tensor(x), torch.as_tensor(y))


def test_install_rebinds_and_restores_keypoint_inference():
    orig_kri, orig_h2k = roi_heads.keypointrcnn_inference, roi_heads.heatmaps_to_keypoints
    vision_b200.install()
    try:
        assert roi_heads.keypointrcnn_inference is not orig_kri and roi_heads.keypointrcnn_inference.__wrapped__ is orig_kri
        assert roi_heads.heatmaps_to_keypoints is not orig_h2k and roi_heads.heatmaps_to_keypoints.__wrapped__ is orig_h2k
    finally:
        vision_b200.uninstall()
    assert roi_heads.keypointrcnn_inference is orig_kri and roi_heads.heatmaps_to_keypoints is orig_h2k


def _refuse(*a, **k):
    raise AssertionError("the fused path must not be taken for these inputs")


def _cases():
    yield "cpu", _inputs()
    yield "fp64_maps", _seen_as_cuda(*_inputs(maps_dtype=torch.float64))
    yield "fp16_rois", _seen_as_cuda(*_inputs(rois_dtype=torch.float16))
    yield "oversized_plane", _seen_as_cuda(*_inputs(H=det.KEYPOINTS_MAX_SIDE + 1, W=6))
    maps, rois = _inputs()
    rois[1, 2] = float("nan")
    yield "nan_box", _seen_as_cuda(maps, rois)


@pytest.mark.parametrize("label", [c[0] for c in _cases()])
def test_uncovered_inputs_take_the_reference_body(label, monkeypatch):
    maps, rois = next(c for c in _cases() if c[0] == label)[1]
    try:
        expected = roi_heads.heatmaps_to_keypoints(maps, rois)
    except ValueError as e:          # a NaN box: int(nan) in the reference loop
        expected = e
    monkeypatch.setattr(det, "heatmaps_to_keypoints_op", _refuse)
    vision_b200.install()
    try:
        if isinstance(expected, Exception):
            with pytest.raises(type(expected), match=str(expected)):
                roi_heads.heatmaps_to_keypoints(maps, rois)
            return
        got = roi_heads.heatmaps_to_keypoints(maps, rois)
        got_kri = roi_heads.keypointrcnn_inference(maps, [rois[:1], rois[1:]])
    finally:
        vision_b200.uninstall()
    _same(got, expected)
    _same(got_kri, roi_heads.keypointrcnn_inference(maps, [rois[:1], rois[1:]]))


def test_tracing_takes_the_reference_onnx_loop(monkeypatch):
    maps, rois = _seen_as_cuda(*_inputs())
    monkeypatch.setattr(tv, "_is_tracing", lambda: True)
    expected = roi_heads.heatmaps_to_keypoints(maps, rois)
    monkeypatch.setattr(det, "heatmaps_to_keypoints_op", _refuse)
    vision_b200.install()
    try:
        got = roi_heads.heatmaps_to_keypoints(maps, rois)
    finally:
        vision_b200.uninstall()
    _same(got, expected)


def test_covered_inputs_take_one_fused_call(monkeypatch):
    """The control for the cases above: the same stand-in inputs in fp32 reach the op, once for all images."""
    maps, rois = _seen_as_cuda(*_inputs(K=5))
    calls = []

    def fused(m, r):
        calls.append(r.shape[0])
        return torch.zeros(r.shape[0], 3, m.shape[1]).permute(0, 2, 1), torch.zeros(r.shape[0], m.shape[1])

    monkeypatch.setattr(det, "heatmaps_to_keypoints_op", fused)
    vision_b200.install()
    try:
        xy, scores = roi_heads.keypointrcnn_inference(maps, [rois[:2], rois[2:2], rois[2:]])
        roi_heads.heatmaps_to_keypoints(maps, rois)
    finally:
        vision_b200.uninstall()
    assert calls == [5, 5]
    assert [t.shape[0] for t in xy] == [2, 0, 3] and [t.shape[0] for t in scores] == [2, 0, 3]


def test_keypoints_workspace_query_needs_no_gpu():
    from vision_b200 import _lib

    q = _lib.core().vb200_heatmaps_to_keypoints_workspace_bytes
    q.restype = ctypes.c_size_t
    assert q(ctypes.c_int64(0), 17) == 0
    one, thousand = q(ctypes.c_int64(1), 17), q(ctypes.c_int64(1000), 17)
    assert 0 < one < thousand
    # per RoI: its geometry, its tile offset and 17 argmax keys; nothing that grows with the resized maps
    assert thousand < 1000 * (16 + 8 + 17 * 8) + 3 * 256
