"""CPU suite: GeneralizedRCNNTransform.forward / .postprocess are rebound by install() and restored by uninstall(); inputs the
fused path does not cover keep running the reference body; the host output-size rule equals the reference's."""
import re

import pytest
import torch

tv = pytest.importorskip("torchvision")
from torchvision.models.detection import transform as tv_transform  # noqa: E402
from torchvision.models.detection.transform import GeneralizedRCNNTransform, _resize_image_and_masks  # noqa: E402

import vision_b200  # noqa: E402
from vision_b200 import detection as det  # noqa: E402

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
KEYPOINT_MIN_SIZES = (640, 672, 704, 736, 768, 800)


class _SeenAsCuda(torch.Tensor):
    """A CPU tensor the coverage predicate takes for a CUDA one, so that each case below is refused for its own reason
    and the reference body can still run here."""

    @property
    def is_cuda(self):
        return True


def _transform(**kw):
    args = dict(min_size=800, max_size=1333, image_mean=MEAN, image_std=STD)
    args.update(kw)
    return GeneralizedRCNNTransform(**args).eval()


def _images(shapes=((3, 48, 64), (3, 40, 30)), dtype=torch.float32, seed=0):
    gen = torch.Generator().manual_seed(seed)
    return [torch.rand(s, generator=gen).to(dtype) for s in shapes]


def _same(a, b):
    if isinstance(a, tv_transform.ImageList):
        assert a.image_sizes == b.image_sizes
        return _same(a.tensors, b.tensors)
    if isinstance(a, (list, tuple)):
        assert type(a) is type(b) and len(a) == len(b)
        for x, y in zip(a, b):
            _same(x, y)
        return
    if isinstance(a, dict):
        assert list(a) == list(b)
        for k in a:
            _same(a[k], b[k])
        return
    if isinstance(a, torch.Tensor):
        assert a.dtype == b.dtype and a.shape == b.shape and a.stride() == b.stride()
        assert torch.equal(a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8))
        return
    assert a == b


def test_install_rebinds_and_restores_the_transform():
    cls = GeneralizedRCNNTransform
    orig_fwd, orig_post = cls.forward, cls.postprocess
    vision_b200.install()
    try:
        assert cls.forward is not orig_fwd and cls.forward.__wrapped__ is orig_fwd
        assert cls.postprocess is not orig_post and cls.postprocess.__wrapped__ is orig_post
    finally:
        vision_b200.uninstall()
    assert cls.forward is orig_fwd and cls.postprocess is orig_post


def _result(n_boxes=(3, 0), keypoints=True, seed=1):
    gen = torch.Generator().manual_seed(seed)
    out = []
    for n in n_boxes:
        xy = torch.rand(n, 2, generator=gen) * 500
        d = {"boxes": torch.cat([xy, xy + torch.rand(n, 2, generator=gen) * 300], 1), "scores": torch.rand(n, generator=gen),
             "labels": torch.ones(n, dtype=torch.int64)}
        if keypoints:
            d["keypoints"] = torch.rand(n, 3, 17, generator=gen).permute(0, 2, 1) * 600
        out.append(d)
    return out


def _clone(result):
    return [{k: v.clone() for k, v in d.items()} for d in result]


def test_cpu_images_match_the_uninstalled_transform():
    t = _transform()
    images = _images()
    want = t(images)
    shapes, orig = [(800, 1066), (800, 600)], [(48, 64), (40, 30)]
    want_post = t.postprocess(_clone(_result()), shapes, orig)
    vision_b200.install()
    try:
        got = t(images)
        got_post = t.postprocess(_clone(_result()), shapes, orig)
    finally:
        vision_b200.uninstall()
    _same(got, want)
    _same(got_post, want_post)


@pytest.mark.parametrize("min_size,max_size,fixed_size", [(800, 1333, None), (KEYPOINT_MIN_SIZES, 1333, None), (300, 300, (300, 300)),
                                                          (320, 320, (320, 320))])
def test_output_size_rule_matches_the_reference(min_size, max_size, fixed_size):
    t = _transform(min_size=min_size, max_size=max_size, fixed_size=fixed_size)
    gen = torch.Generator().manual_seed(0)
    hs = torch.cat([torch.randint(1, 4000, (1500,), generator=gen), torch.arange(1, 300)])
    ws = torch.cat([torch.randint(1, 4000, (1500,), generator=gen), torch.arange(300, 1, -1)])
    for h, w in zip(hs.tolist(), ws.tolist()):
        ref, _ = _resize_image_and_masks(torch.empty(3, h, w, device="meta"), t.min_size[-1], t.max_size, None, t.fixed_size)
        assert det.rcnn_output_size(h, w, t.min_size[-1], t.max_size, t.fixed_size) == tuple(ref.shape[-2:]), (h, w)


def _refuse(*a, **k):
    raise AssertionError("the fused path must not be taken for these inputs")


def _seen_as_cuda(images):
    return [img.as_subclass(_SeenAsCuda) for img in images]


def _forward_cases():
    yield "training", _transform().train(), _seen_as_cuda(_images()), None
    yield "targets", _transform(), _seen_as_cuda(_images()), [{"boxes": torch.tensor([[1.0, 2.0, 10.0, 12.0]])}] * 2
    yield "fp64", _transform(), _seen_as_cuda(_images(dtype=torch.float64)), None
    yield "uint8", _transform(), _seen_as_cuda([(img * 255).to(torch.uint8) for img in _images()]), None
    yield "mixed_dtypes", _transform(), _seen_as_cuda([_images()[0], _images()[1].half()]), None
    yield "mean_broadcast", _transform(image_mean=[0.5], image_std=[0.25]), _seen_as_cuda(_images()), None
    yield "nine_channels", _transform(image_mean=[0.5] * 9, image_std=[0.25] * 9), _seen_as_cuda(_images(((9, 20, 30),))), None
    yield "mixed_channels", _transform(image_mean=[0.5], image_std=[0.25]), _seen_as_cuda(_images(((1, 20, 30), (3, 20, 30)))), None
    yield "empty_output", _transform(min_size=1, max_size=1), _seen_as_cuda(_images(((3, 10, 400),))), None
    yield "two_dim_image", _transform(), _seen_as_cuda([torch.rand(20, 30)]), None


@pytest.mark.parametrize("label", [c[0] for c in _forward_cases()])
def test_uncovered_inputs_take_the_reference_forward(label, monkeypatch):
    _, t, images, targets = next(c for c in _forward_cases() if c[0] == label)
    try:
        want = t(images, targets)
    except (TypeError, ValueError, RuntimeError) as e:
        want = e
    monkeypatch.setattr(det, "rcnn_batch_images_op", _refuse)
    vision_b200.install()
    try:
        if isinstance(want, Exception):
            with pytest.raises(type(want), match=re.escape(str(want).splitlines()[0])):
                t(images, targets)
            return
        got = t(images, targets)
    finally:
        vision_b200.uninstall()
    _same(got, want)


def test_deterministic_mode_and_tracing_take_the_reference_forward(monkeypatch):
    t, images = _transform(), _seen_as_cuda(_images())
    torch.use_deterministic_algorithms(True)
    try:
        want_det = t(images)
    finally:
        torch.use_deterministic_algorithms(False)
    want = t(images)
    monkeypatch.setattr(det, "rcnn_batch_images_op", _refuse)
    vision_b200.install()
    try:
        torch.use_deterministic_algorithms(True)
        try:
            got_det = t(images)
        finally:
            torch.use_deterministic_algorithms(False)
        monkeypatch.setattr(det, "_traced", lambda: True)
        got_traced = t(images)
    finally:
        vision_b200.uninstall()
    _same(got_det, want_det)
    _same(got_traced, want)


def test_covered_inputs_take_one_fused_call(monkeypatch):
    """The control for the cases above: stand-in fp32 images of a 4-D batch reach the op once, with the reference's sizes,
    padding and mean / std rounded to the images' dtype."""
    t = _transform(size_divisible=32)
    calls = []

    def fused(images, sizes, pad_h, pad_w, mean, std):
        calls.append((len(images), list(sizes), pad_h, pad_w, mean, std))
        return torch.zeros(len(images), 3, pad_h, pad_w)

    monkeypatch.setattr(det, "rcnn_batch_images_op", fused)
    batch = torch.rand(2, 3, 480, 640).as_subclass(_SeenAsCuda)
    vision_b200.install()
    try:
        image_list, targets = t(batch)
        t(_seen_as_cuda(_images(dtype=torch.float16)))
    finally:
        vision_b200.uninstall()
    assert targets is None and image_list.image_sizes == [(800, 1066), (800, 1066)]
    assert all(type(v) is int for hw in image_list.image_sizes for v in hw)
    assert calls[0] == (2, [(800, 1066)] * 2, 800, 1088, torch.tensor(MEAN).tolist(), torch.tensor(STD).tolist())
    assert calls[1][4] == torch.tensor(MEAN, dtype=torch.float16).tolist() != torch.tensor(MEAN).tolist()


def test_postprocess_takes_one_fused_call(monkeypatch):
    t = _transform()
    calls = []

    def fused(inputs, rw, rh):
        calls.append((len(inputs), list(rw), list(rh)))
        return [torch.zeros(x.shape[0], 4) if x.dim() == 2 else torch.empty_like(x) for x in inputs]

    monkeypatch.setattr(det, "rcnn_rescale_op", fused)
    result = [{k: v.as_subclass(_SeenAsCuda) if v.is_floating_point() else v for k, v in d.items()} for d in _result()]
    vision_b200.install()
    try:
        t.postprocess(result, [(800, 1066), (800, 600)], [(480, 640), (427, 320)])
    finally:
        vision_b200.uninstall()
    f32 = lambda a, b: float(torch.tensor(a, dtype=torch.float32) / torch.tensor(b, dtype=torch.float32))  # noqa: E731
    assert calls == [(4, [f32(640, 1066)] * 2 + [f32(320, 600)] * 2, [f32(480, 800)] * 2 + [f32(427, 800)] * 2)]


def test_uncovered_results_take_the_reference_postprocess(monkeypatch):
    t = _transform()
    shapes, orig = [(800, 1066), (800, 600)], [(480, 640), (427, 320)]
    monkeypatch.setattr(det, "rcnn_rescale_op", _refuse)
    for result in (_result(),                                                        # CPU tensors
                   [{k: v.double() if v.is_floating_point() else v for k, v in d.items()} for d in _result()]):
        want = t.postprocess(_clone(result), shapes, orig)
        seen = [{k: v.as_subclass(_SeenAsCuda) if v.dtype == torch.float64 else v for k, v in d.items()} for d in _clone(result)]
        vision_b200.install()
        try:
            got = t.postprocess(seen, shapes, orig)
        finally:
            vision_b200.uninstall()
        _same(got, want)
