"""GPU suite: Keypoint R-CNN's heatmaps_to_keypoints / keypointrcnn_inference through install() against the same functions
with vision_b200 uninstalled (torchvision's own loop over F.interpolate and argmax), bit for bit, with the reference's
shapes and strides, and with the keypoint kernels counted as launched."""
import pytest
import torch

tv = pytest.importorskip("torchvision")
from torchvision.models.detection import roi_heads  # noqa: E402

pytestmark = pytest.mark.gpu

N_KP, SIDE = 17, 56


def _rois(K, seed=0, max_w=1333.0, max_h=800.0):
    """Boxes of every size class the reference treats differently: sub-pixel (clamped to 1), x2 < x1, downscale (< 56),
    exactly 56 x 56 (the same-size copy), integer and fractional edges, and up to max_w x max_h."""
    gen = torch.Generator().manual_seed(seed)
    x1 = torch.rand(K, generator=gen) * 1000 - 50
    y1 = torch.rand(K, generator=gen) * 700 - 50
    w = torch.rand(K, generator=gen) * max_w
    h = torch.rand(K, generator=gen) * max_h
    kind = torch.arange(K) % 7
    w = torch.where(kind == 0, torch.rand(K, generator=gen) * 0.9, w)
    h = torch.where(kind == 0, torch.rand(K, generator=gen) * 0.9, h)
    w = torch.where(kind == 1, -torch.rand(K, generator=gen) * 20, w)
    w = torch.where(kind == 2, torch.rand(K, generator=gen) * 55, w)
    h = torch.where(kind == 2, torch.rand(K, generator=gen) * 55, h)
    w = torch.where(kind == 3, 55.0 + torch.rand(K, generator=gen), w)          # ceil(w) == ceil(h) == 56: the copy case
    h = torch.where(kind == 3, 55.0 + torch.rand(K, generator=gen), h)
    x1 = torch.where(kind == 4, x1.round(), x1)
    y1 = torch.where(kind == 4, y1.round(), y1)
    w = torch.where(kind == 4, w.round(), w)
    h = torch.where(kind == 4, h.round(), h)
    w = torch.where(kind == 5, torch.full((K,), max_w), w)
    h = torch.where(kind == 5, torch.full((K,), max_h), h)
    boxes = torch.stack([x1, y1, x1 + w, y1 + h], 1)
    return boxes.cuda()


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _same(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        if isinstance(w, (list, tuple)):
            _same(g, w)
            continue
        assert g.dtype == w.dtype and g.shape == w.shape and g.stride() == w.stride() and g.device == w.device
        assert torch.equal(_bits(g), _bits(w)), (g - w).abs().nan_to_num(0).max()


def _fused(vb, fn):
    """fn() through install() (fn looks the rebound globals up when it runs), with the number of vision_b200 launches it made."""
    vb.install()
    try:
        before = vb.launch_count()
        out = fn()
        torch.cuda.synchronize()
        return out, vb.launch_count() - before
    finally:
        vb.uninstall()


def _check(vb, maps, rois):
    assert not vb.installed()
    want = roi_heads.heatmaps_to_keypoints(maps, rois)
    got, launches = _fused(vb, lambda: roi_heads.heatmaps_to_keypoints(maps, rois))
    _same(got, want)
    assert launches == (3 if rois.shape[0] else 0)
    return launches


@pytest.mark.parametrize("K", [0, 1, 100, 1000])
def test_heatmaps_to_keypoints_matches_reference(vb, K):
    gen = torch.Generator(device="cuda").manual_seed(K)
    maps = torch.randn(K, N_KP, SIDE, SIDE, generator=gen, device="cuda")
    _check(vb, maps, _rois(K, seed=K))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_precision_maps(vb, dtype):
    gen = torch.Generator(device="cuda").manual_seed(1)
    maps = (torch.randn(140, N_KP, SIDE, SIDE, generator=gen, device="cuda") * 3).to(dtype)
    _check(vb, maps, _rois(140, seed=1))


@pytest.mark.parametrize("levels", [1, 3])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_ties(vb, levels, dtype):
    """Constant maps and maps of a few levels: many equal maxima, the lowest flat index must win."""
    gen = torch.Generator(device="cuda").manual_seed(2)
    maps = torch.randint(0, levels, (70, N_KP, SIDE, SIDE), generator=gen, device="cuda").to(dtype) * 0.5
    _check(vb, maps, _rois(70, seed=2, max_w=300.0, max_h=300.0))


def test_non_finite_and_signed_zero_maps(vb):
    gen = torch.Generator(device="cuda").manual_seed(3)
    K = 70
    maps = torch.randn(K, N_KP, SIDE, SIDE, generator=gen, device="cuda")
    flat = maps.view(-1)
    n = flat.numel()
    for value, count in ((float("nan"), 400), (float("inf"), 400), (float("-inf"), 400), (-0.0, 400)):
        flat[torch.randint(0, n, (count,), generator=gen, device="cuda")] = value
    maps[0::7, :3] = -0.0                          # whole maps of -0.0 and +0.0, in every size class
    maps[1::7, 3:6] = 0.0
    maps[2::7, 6, 0, 0] = float("inf")             # an inf in a corner
    maps[3::7, 7, -1, -1] = float("-inf")
    maps[4::7, 8] = float("-inf")                  # a whole map of -inf
    _check(vb, maps, _rois(K, seed=3, max_w=400.0, max_h=300.0))


def test_non_contiguous_maps(vb):
    gen = torch.Generator(device="cuda").manual_seed(4)
    maps = torch.randn(60, SIDE, N_KP, SIDE, generator=gen, device="cuda").permute(0, 2, 1, 3)
    assert not maps.is_contiguous()
    _check(vb, maps, _rois(60, seed=4, max_w=500.0, max_h=500.0))


@pytest.mark.parametrize("counts", [[7], [5, 0], [3, 9, 0, 1, 12, 4, 6, 2]])
def test_keypointrcnn_inference_one_call_for_all_images(vb, counts):
    gen = torch.Generator(device="cuda").manual_seed(len(counts))
    x = torch.randn(sum(counts), N_KP, SIDE, SIDE, generator=gen, device="cuda")
    boxes = list(_rois(sum(counts), seed=5, max_w=600.0, max_h=600.0).split(counts))
    want = roi_heads.keypointrcnn_inference(x, boxes)
    got, launches = _fused(vb, lambda: roi_heads.keypointrcnn_inference(x, boxes))
    _same(got, want)
    assert launches == 3


def test_non_finite_boxes_raise_the_reference_error(vb):
    maps = torch.randn(4, N_KP, SIDE, SIDE, device="cuda")
    for bad in (float("nan"), float("inf")):
        rois = _rois(4, seed=6)
        rois[2, 2] = bad
        with pytest.raises((ValueError, OverflowError)) as want:
            roi_heads.heatmaps_to_keypoints(maps, rois)
        vb.install()
        try:
            with pytest.raises(want.type, match=str(want.value)):
                roi_heads.heatmaps_to_keypoints(maps, rois)
        finally:
            vb.uninstall()


def test_launch_count_does_not_grow_with_rois(vb):
    gen = torch.Generator(device="cuda").manual_seed(7)
    counts = []
    for K in (1, 1000):
        maps = torch.randn(K, N_KP, SIDE, SIDE, generator=gen, device="cuda")
        rois = _rois(K, seed=7, max_w=200.0, max_h=200.0)
        counts.append(_fused(vb, lambda: roi_heads.heatmaps_to_keypoints(maps, rois))[1])
    assert counts[0] == counts[1] == 3


def test_keypoint_rcnn_end_to_end(vb, monkeypatch):
    """A Keypoint R-CNN forward with install(), against the same forward with only the two keypoint globals put back.
    The rest of the model is held on the installed path in both runs: the installed roi_align follows the reference's CPU
    arithmetic, a few ulps away from its CUDA kernel, so the boxes, and the keypoints with them, would differ for that
    reason alone."""
    from torchvision.models.detection import keypointrcnn_resnet50_fpn

    from vision_b200 import detection as det

    torch.manual_seed(0)
    model = keypointrcnn_resnet50_fpn(weights=None, weights_backbone=None, box_score_thresh=0.0).cuda().eval()
    gen = torch.Generator(device="cuda").manual_seed(8)
    images = [torch.rand(3, 480, 640, generator=gen, device="cuda"), torch.rand(3, 512, 384, generator=gen, device="cuda")]
    calls = []
    op = det.heatmaps_to_keypoints_op
    monkeypatch.setattr(det, "heatmaps_to_keypoints_op", lambda maps, rois: calls.append(rois.shape[0]) or op(maps, rois))
    originals = roi_heads.keypointrcnn_inference, roi_heads.heatmaps_to_keypoints
    deterministic = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    vb.install()
    try:
        with torch.no_grad():
            got = model(images)
            roi_heads.keypointrcnn_inference, roi_heads.heatmaps_to_keypoints = originals
            want = model(images)
    finally:
        vb.uninstall()
        torch.backends.cudnn.deterministic = deterministic
    assert roi_heads.keypointrcnn_inference is originals[0]
    detections = [int(w["keypoints"].shape[0]) for w in want]
    assert sum(detections) > 0 and calls == [sum(detections)]          # one fused call for both images
    for g, w in zip(got, want):
        assert torch.equal(g["boxes"], w["boxes"])
        _same([g["keypoints"], g["keypoints_scores"]], [w["keypoints"], w["keypoints_scores"]])
