"""GPU suite: GeneralizedRCNNTransform.forward / .postprocess through install() against the same calls with vision_b200
uninstalled (torchvision's per-image normalize, F.interpolate and batch_images; resize_boxes / resize_keypoints), bit for
bit, with the reference's dtypes, shapes and strides, one vision_b200 launch per call and no host synchronisation."""
import pytest
import torch

tv = pytest.importorskip("torchvision")
from torchvision.models.detection.transform import GeneralizedRCNNTransform  # noqa: E402

from vision_b200 import detection as det  # noqa: E402

pytestmark = pytest.mark.gpu

IMAGENET = dict(image_mean=[0.485, 0.456, 0.406], image_std=[0.229, 0.224, 0.225])
CONFIGS = {   # the settings torchvision's detection builders pass (faster_rcnn.py, keypoint_rcnn.py, ssd.py, ssdlite.py)
    "faster_rcnn": dict(min_size=800, max_size=1333, **IMAGENET),
    "keypoint_rcnn": dict(min_size=(640, 672, 704, 736, 768, 800), max_size=1333, **IMAGENET),
    "ssd300": dict(min_size=300, max_size=300, image_mean=[0.48235, 0.45882, 0.40784], image_std=[1.0 / 255.0] * 3, size_divisible=1,
                   fixed_size=(300, 300)),
    "ssdlite": dict(min_size=320, max_size=320, image_mean=[0.5] * 3, image_std=[0.5] * 3, size_divisible=1, fixed_size=(320, 320)),
}
# 800 x 1067 and 800 x 1333 keep their size under (800, 1333); 300 x 1200 is capped by max_size; 17 x 23 is a x47 upscale
SHAPES = [(480, 640), (427, 640), (640, 480), (300, 1200), (17, 23), (3000, 2000), (800, 1067), (800, 1333)]
BATCHES = {1: SHAPES[:1], 2: SHAPES[1:3], 8: SHAPES}


def _transform(name="faster_rcnn", **kw):
    return GeneralizedRCNNTransform(**{**CONFIGS[name], **kw}).eval()


def _images(shapes, dtype=torch.float32, dist="uniform", C=3, seed=0):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    draw = torch.rand if dist == "uniform" else torch.randn
    return [draw(C, h, w, generator=gen, device="cuda").to(dtype) for h, w in shapes]


def _bits(t):
    return t.reshape(-1).view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _same(got, want):
    if isinstance(want, (list, tuple)):
        assert type(got) is type(want) and len(got) == len(want)
        for g, w in zip(got, want):
            _same(g, w)
    elif isinstance(want, dict):
        assert list(got) == list(want)
        for k in want:
            _same(got[k], want[k])
    elif isinstance(want, torch.Tensor):
        assert got.dtype == want.dtype and got.shape == want.shape and got.stride() == want.stride() and got.device == want.device
        diff = _bits(got) != _bits(want)
        assert not diff.any(), f"{int(diff.sum())} elements differ" + (
            f", per leading index {diff.view(got.shape).flatten(1).sum(1).tolist()}" if got.dim() > 1 and got.numel() else "")
    elif hasattr(want, "image_sizes"):
        assert got.image_sizes == want.image_sizes
        assert all(type(v) is int for hw in got.image_sizes for v in hw)
        _same(got.tensors, want.tensors)
    else:
        assert got == want


def _installed(vb, fn):
    """fn() through install(), with the number of vision_b200 launches it made."""
    vb.install()
    try:
        before = vb.launch_count()
        out = fn()
        torch.cuda.synchronize()
        return out, vb.launch_count() - before
    finally:
        vb.uninstall()


def _check_forward(vb, t, images, launches=1):
    assert not vb.installed()
    want = t(images)
    got, n = _installed(vb, lambda: t(images))
    _same(got, want)
    assert n == launches
    return got


@pytest.mark.parametrize("dist", ["uniform", "normal"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("batch", sorted(BATCHES))
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_forward_matches_reference(vb, name, batch, dtype, dist):
    _check_forward(vb, _transform(name), _images(BATCHES[batch], dtype, dist, seed=batch))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_one_channel(vb, dtype):
    t = _transform(image_mean=[0.45], image_std=[0.226])
    _check_forward(vb, t, _images(BATCHES[8], dtype, "normal", C=1))


def test_four_dim_batch(vb):
    gen = torch.Generator(device="cuda").manual_seed(1)
    _check_forward(vb, _transform(), torch.rand(2, 3, 480, 640, generator=gen, device="cuda"))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_non_finite_pixels(vb, dtype):
    """inf and NaN in a resized image and in a same-size one (800 x 1067): the bilinear taps that meet them with weight 0
    decide whether they spread."""
    images = _images([(480, 640), (800, 1067), (800, 1333)], dtype, "normal", seed=2)
    gen = torch.Generator(device="cuda").manual_seed(3)
    for img in images[:2]:
        flat = img.view(-1)
        for value in (float("inf"), float("-inf"), float("nan")):
            flat[torch.randint(0, flat.numel(), (50,), generator=gen, device="cuda")] = value
    images[1][:, 0, -1] = float("inf")               # last column and last row: taps clamped to the edge
    images[1][:, -1, 5] = float("nan")
    _check_forward(vb, _transform(), images)


def test_strided_inputs(vb):
    """An HWC array permuted to CHW (the reference takes ATen's channels-last kernel) and a cropped view, read in place."""
    gen = torch.Generator(device="cuda").manual_seed(4)
    hwc = torch.rand(480, 640, 3, generator=gen, device="cuda").permute(2, 0, 1)
    big = torch.randn(3, 700, 900, generator=gen, device="cuda")
    crop = big[:, 13:440, 21:661]
    hwc_half = torch.rand(427, 640, 3, generator=gen, device="cuda").half().permute(2, 0, 1)
    for t in (_transform(), _transform("ssd300")):
        _check_forward(vb, t, [hwc, crop])
        _check_forward(vb, t, [hwc_half])


def test_fasterrcnn_model_takes_the_fused_transform(vb, monkeypatch):
    from torchvision.models.detection import fasterrcnn_resnet50_fpn

    transform = fasterrcnn_resnet50_fpn(weights=None, weights_backbone=None).eval().cuda().transform
    calls = []
    op = det.rcnn_batch_images_op
    monkeypatch.setattr(det, "rcnn_batch_images_op", lambda *a: calls.append(len(a[0])) or op(*a))
    _check_forward(vb, transform, _images(BATCHES[2], seed=5))
    assert calls == [2]


def _result(counts, keypoints=None, masks=False, seed=6):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for n in counts:
        xy = torch.rand(n, 2, generator=gen, device="cuda") * 500       # boxes inside every image: masks are pasted into them
        d = {"boxes": torch.cat([xy, xy + torch.rand(n, 2, generator=gen, device="cuda") * 250], 1),
             "labels": torch.ones(n, dtype=torch.int64, device="cuda"), "scores": torch.rand(n, generator=gen, device="cuda")}
        if keypoints == "contiguous":
            d["keypoints"] = torch.rand(n, 17, 3, generator=gen, device="cuda") * 1000
        elif keypoints == "permuted":      # the fused keypoint path's views of a [K, 3, 17] buffer
            d["keypoints"] = (torch.rand(n, 3, 17, generator=gen, device="cuda") * 1000).permute(0, 2, 1)
            d["keypoints_scores"] = torch.rand(n, 17, generator=gen, device="cuda")
        if masks:
            d["masks"] = torch.rand(n, 1, 28, 28, generator=gen, device="cuda")
        out.append(d)
    return out


def _clone(result):
    return [{k: v.clone(memory_format=torch.preserve_format) for k, v in d.items()} for d in result]


def _check_postprocess(vb, t, result, image_shapes, original_sizes, launches=1):
    want = t.postprocess(_clone(result), image_shapes, original_sizes)
    got, n = _installed(vb, lambda: t.postprocess(_clone(result), image_shapes, original_sizes))
    _same(got, want)
    assert n == launches


SIZES = {"shapes": [(800, 1066), (800, 1201), (800, 1066)], "orig": [(480, 640), (533, 800), (427, 569)]}


@pytest.mark.parametrize("keypoints", [None, "contiguous", "permuted"])
@pytest.mark.parametrize("counts", [[0], [100], [100, 0, 37]])
def test_postprocess_matches_reference(vb, counts, keypoints):
    n = len(counts)
    _check_postprocess(vb, _transform(), _result(counts, keypoints), SIZES["shapes"][:n], SIZES["orig"][:n])


def test_postprocess_with_masks(vb):
    _check_postprocess(vb, _transform(), _result([20, 5], masks=True), SIZES["shapes"][:2], SIZES["orig"][:2])


def test_forward_and_postprocess_do_not_synchronize(vb):
    t = _transform("keypoint_rcnn")
    images = _images(BATCHES[8], seed=7)
    result = _result([100] * 8, "permuted")
    vb.install()
    try:
        torch.cuda.set_sync_debug_mode("error")
        try:
            image_list, _ = t(images)
            t.postprocess(result, image_list.image_sizes, [tuple(img.shape[-2:]) for img in images])
        finally:
            torch.cuda.set_sync_debug_mode(0)
    finally:
        vb.uninstall()


FORWARD_FALLBACKS = ["training", "targets", "fp64", "uint8", "mixed_dtypes", "mixed_devices", "cpu", "mean_broadcast", "nine_channels",
                     "empty_output"]


def _forward_fallback(label):
    imgs = lambda dtype=torch.float32, C=3: _images(BATCHES[2], dtype, C=C, seed=8)  # noqa: E731
    return {
        "training": lambda: (_transform().train(), imgs(), None),
        "targets": lambda: (_transform(), imgs(), [{"boxes": torch.tensor([[1.0, 2.0, 30.0, 40.0]], device="cuda")}] * 2),
        "fp64": lambda: (_transform(), imgs(torch.float64), None),
        "uint8": lambda: (_transform(), [(img * 255).to(torch.uint8) for img in imgs()], None),
        "mixed_dtypes": lambda: (_transform(), [imgs()[0], imgs(torch.float16)[1]], None),
        "mixed_devices": lambda: (_transform(), [imgs()[0], imgs()[1].cpu()], None),
        "cpu": lambda: (_transform(), [img.cpu() for img in imgs()], None),
        "mean_broadcast": lambda: (_transform(image_mean=[0.5], image_std=[0.25]), imgs(), None),
        "nine_channels": lambda: (_transform(image_mean=[0.5] * 9, image_std=[0.25] * 9), imgs(C=9), None),
        "empty_output": lambda: (_transform(min_size=1, max_size=1), _images([(10, 400)]), None),
    }[label]()


@pytest.mark.parametrize("label", FORWARD_FALLBACKS)
def test_forward_fallbacks_run_the_reference(vb, label):
    t, images, targets = _forward_fallback(label)
    torch.manual_seed(0)
    try:
        want = t(images, targets)
    except (TypeError, ValueError, RuntimeError) as e:
        want = e
    vb.install()
    try:
        before = vb.launch_count()
        torch.manual_seed(0)
        if isinstance(want, Exception):
            with pytest.raises(type(want)):
                t(images, targets)
        else:
            got = t(images, targets)
            _same(got, want)
        assert vb.launch_count() == before
    finally:
        vb.uninstall()


def test_deterministic_mode_and_autocast_run_the_reference(vb):
    t = _transform()
    for dtype, mode in ((torch.float32, "deterministic"), (torch.float16, "autocast"), (torch.bfloat16, "autocast")):
        images = _images(BATCHES[2], dtype, seed=9)

        def run():
            if mode == "deterministic":
                torch.use_deterministic_algorithms(True)
                try:
                    return t(images)
                finally:
                    torch.use_deterministic_algorithms(False)
            with torch.autocast("cuda", dtype=torch.float16):
                return t(images)

        want = run()
        got, n = _installed(vb, run)
        _same(got, want)
        assert n == 0, mode


def test_postprocess_fallbacks_run_the_reference(vb):
    t = _transform()
    half = [{k: v.half() if v.is_floating_point() else v for k, v in d.items()} for d in _result([10, 3])]
    _check_postprocess(vb, t, half, SIZES["shapes"][:2], SIZES["orig"][:2], launches=0)
    _check_postprocess(vb, t.train(), _result([10, 3]), SIZES["shapes"][:2], SIZES["orig"][:2], launches=0)
