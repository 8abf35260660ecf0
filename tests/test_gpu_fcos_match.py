"""GPU suite: FCOS's fused training-target assignment against the reference on the same GPU, bit for bit.  Each case calls
FCOS.compute_loss (with a head that returns the matched indices) uninstalled and installed on the same inputs and compares
values, dtype, shape, stride and device; one training step of fcos_resnet50_fpn compares full install() with install()
minus the FCOS rebind."""
import math
import types

import pytest
import torch

tv = pytest.importorskip("torchvision")
from torchvision.models.detection import fcos  # noqa: E402

import vision_b200  # noqa: E402

pytestmark = pytest.mark.gpu

STRIDES = (8, 16, 32, 64, 128)
# padded batch sizes of images in one call: different N per image (18,134 anchors for 800 x 1088)
SIDES = [(800, 1088), (640, 800), (512, 704), (800, 800), (320, 448), (768, 1024), (608, 608), (416, 640)]
DTYPE_PAIRS = [(torch.float32, torch.float32), (torch.float16, torch.float32), (torch.bfloat16, torch.float32),
               (torch.float32, torch.float16), (torch.float16, torch.float16), (torch.float32, torch.bfloat16),
               (torch.float64, torch.float64)]          # (anchors, gt)


def _anchors(h, w):
    """FCOS's anchors of an h x w batch: one stride-sized box per location and level, level by level."""
    per_level = []
    for s in STRIDES:
        ys, xs = torch.meshgrid(torch.arange(-(-h // s)) * s, torch.arange(-(-w // s)) * s, indexing="ij")
        xy = torch.stack([xs.reshape(-1), ys.reshape(-1)], 1).float()
        per_level.append(torch.cat([xy - s / 2, xy + s / 2], 1))
    return torch.cat(per_level).cuda(), [p.shape[0] for p in per_level]


def _gt(M, gen, h, w):
    """Boxes of 8 to 600 pixels a side (log-uniform), so that every level has gt in its scale range."""
    c = torch.rand(M, 2, generator=gen) * torch.tensor([w, h])
    s = torch.exp(torch.rand(M, 2, generator=gen) * math.log(600 / 8)) * 8
    return torch.cat([c - s / 2, c + s / 2], 1).cuda()


def _problem(M, B, seed=0):
    gen = torch.Generator().manual_seed(seed)
    gts, anchors, levels = [], [], None
    for i in range(B):
        h, w = SIDES[i % len(SIDES)]
        a, lv = _anchors(h, w)
        levels = levels or lv
        anchors.append(a)
        gts.append(_gt(M, gen, h, w))
    return gts, anchors, levels


def _special_problem():
    """Two 800 x 1088 images.  The first one's gt boxes put anchor centres exactly on gt edges, at radius * size from a gt
    centre and at the level bounds (and just inside them), with gt areas that tie under 1e8 - area in fp32, areas of 1e8 and
    above, inverted boxes and duplicates.  The second has NaN and infinite coordinates: their 1e8 - area is NaN or -inf, so
    every anchor that does not match them gets a NaN value, which wins the argmax."""
    a, levels = _anchors(800, 1088)
    gen = torch.Generator().manual_seed(7)
    boxes = [
        [480, 380, 520, 420], [440, 380, 480, 420], [470, 400, 510, 440], [470, 360, 510, 400],   # edges through (480, 400)
        [472, 380, 512, 420], [460, 380, 500, 420], [452, 384, 508, 416],   # centre 12 / 20 from (480, 400): r * 8 at r = 1.5 / 2.5
        [416, 256, 544, 384], [415.5, 255.5, 544.5, 384.5],                 # max distance 64 (= 4 * 16) and 64.5 around (480, 320)
        [352, 192, 608, 448], [352.5, 192.5, 607.5, 447.5],                 # 128 (= 8 * 16) and 127.5 around (480, 320)
        [416, 336, 544, 464],                                               # 64 (= 8 * 8) around (480, 400)
        [300, 300, 340.08, 325], [300, 300, 340.04, 325], [300, 300, 340, 325], [300, 300, 340, 325.01],   # areas near 1000
        [640 - 6000, 384 - 4500, 640 + 6000, 384 + 4500],                   # area 1.08e8 around a last-level anchor
        [640 - 5000, 384 - 5000, 640 + 5000, 384 + 5000],                   # area exactly 1e8
        [520, 420, 480, 380], [600, 200, 560, 260],                         # inverted
    ]
    gt = torch.tensor(boxes, dtype=torch.float32)
    rand = _gt(40, gen, 800, 1088).cpu()
    first = torch.cat([gt, rand, gt[:4], rand[:5]])                         # duplicates after the originals
    odd = torch.tensor([[float("nan"), 380, 520, 420], [460, 380, float("inf"), 420], [-float("inf"), 100, 700, 500]])
    second = torch.cat([rand[:10], odd, rand[10:20]])
    return [first.cuda(), second.cuda()], [a, a.clone()], levels


def _owner(radius=1.5):
    head = types.SimpleNamespace(compute_loss=lambda targets, outputs, anchors, matched: matched)
    return types.SimpleNamespace(center_sampling_radius=radius, head=head)


def _call(gts, anchors, levels, radius=1.5):
    return fcos.FCOS.compute_loss(_owner(radius), [{"boxes": g} for g in gts], {}, anchors, levels)


def _installed(fn):
    vision_b200.install()
    try:
        before = vision_b200.launch_count()
        out = fn()
        torch.cuda.synchronize()
        return out, vision_b200.launch_count() - before
    finally:
        vision_b200.uninstall()


def _same(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.shape == w.shape and g.stride() == w.stride() and g.device == w.device
        assert torch.equal(g, w)


def _check(gts, anchors, levels, radius=1.5):
    want = _call(gts, anchors, levels, radius)
    got, launches = _installed(lambda: _call(gts, anchors, levels, radius))
    _same(got, want)
    assert launches == 1
    return want


@pytest.mark.parametrize("B", [1, 2, 8])
@pytest.mark.parametrize("M", [1, 3, 50, 300])
def test_matches_equal_the_reference(M, B):
    want = _check(*_problem(M, B, seed=M * 10 + B))
    assert any((w >= 0).any() for w in want)          # the problem does match anchors


@pytest.mark.parametrize("radius", [0, 1.3, 1.5, 2.5])
def test_radius(radius):
    _check(*_problem(50, 2, seed=3), radius=radius)
    _check(*_special_problem(), radius=radius)


@pytest.mark.parametrize("radius", [1.5, 2.5])
def test_edges_bounds_area_ties_huge_nan_inf_inverted_and_duplicate_boxes(radius):
    want = _check(*_special_problem(), radius=radius)
    assert (want[0] >= 0).any() and (want[0] == -1).any() and (want[1] >= 0).all()


@pytest.mark.parametrize("anchor_dtype,gt_dtype", DTYPE_PAIRS)
def test_dtypes(anchor_dtype, gt_dtype):
    gts, anchors, levels = _problem(50, 2, seed=5)
    special_gts, special_anchors, _ = _special_problem()
    gts, anchors = gts + special_gts, anchors + special_anchors
    want = _check([g.to(gt_dtype) for g in gts], [x.to(anchor_dtype) for x in anchors], levels)
    if gt_dtype == torch.float16:
        # 1e8 - area is inf in fp16: a non-match is 0 * inf = NaN, so no anchor is ever -1
        assert all((w >= 0).all() for w in want)


@pytest.mark.parametrize("case", ["last_level_empty", "first_level_beyond_n", "both"])
def test_level_sizes(case):
    gts, anchors, levels = _problem(50, 3, seed=9)
    if case in ("last_level_empty", "both"):
        levels = levels[:-1] + [0]          # upper_bound[-0:] = inf: every upper bound is inf
    if case in ("first_level_beyond_n", "both"):
        levels = [10**6] + levels[1:]       # lower_bound[:10**6] = 0: every lower bound is 0
    _check(gts, anchors, levels)


def test_background_images_and_an_image_without_anchors():
    gts, anchors, levels = _problem(7, 5, seed=11)
    gts[1] = torch.zeros(0, 4, device="cuda")
    gts[3] = torch.zeros(0, device="cuda")
    anchors[4] = anchors[4][:0]
    want = _check(gts, anchors, levels)
    assert (want[1] == -1).all() and (want[3] == -1).all() and want[4].numel() == 0


def test_all_background():
    gts, anchors, levels = _problem(3, 3, seed=12)
    _check([torch.zeros(0, 4, device="cuda")] * 3, anchors, levels)


def test_fcos_matching_does_not_sync_the_host():
    gts, anchors, levels = _problem(50, 4, seed=13)
    gts[2] = torch.zeros(0, 4, device="cuda")
    _installed(lambda: _call(gts, anchors, levels))        # loads the ops outside the checked region
    vision_b200.install()
    try:
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            _call(gts, anchors, levels)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    finally:
        vision_b200.uninstall()


def test_launch_count_does_not_grow_with_the_batch():
    counts = []
    for B in (1, 8):
        gts, anchors, levels = _problem(50, B, seed=B)
        counts.append(_installed(lambda: _call(gts, anchors, levels))[1])
    assert counts[0] == counts[1] == 1


# ---- one training step ----------------------------------------------------------------------------------------------------

def _train_step(fused_matching: bool):
    from vision_b200 import _install

    torch.manual_seed(0)
    model = tv.models.detection.fcos_resnet50_fpn(weights=None, weights_backbone=None, num_classes=5, min_size=320,
                                                  max_size=448).cuda().train()
    gen = torch.Generator().manual_seed(1)
    images = [torch.rand(3, 300 + 40 * i, 420 - 30 * i, generator=gen).cuda() for i in range(2)]
    targets = []
    for i, img in enumerate(images):
        h, w = img.shape[1:]
        xy = torch.rand(3 + i, 2, generator=gen) * torch.tensor([w * 0.6, h * 0.6])
        wh = torch.rand(3 + i, 2, generator=gen) * torch.tensor([w * 0.35, h * 0.35]) + 8
        targets.append({"boxes": torch.cat([xy, xy + wh], 1).cuda(), "labels": torch.randint(1, 5, (3 + i,), generator=gen).cuda()})
    key = (fcos.FCOS, "compute_loss")
    fused = fcos.FCOS.compute_loss
    if not fused_matching:
        fcos.FCOS.compute_loss = _install._state["matching"][key]
    try:
        torch.manual_seed(2)
        losses = model(images, targets)
        sum(losses.values()).backward()
    finally:
        fcos.FCOS.compute_loss = fused
    torch.cuda.synchronize()
    return {k: v.detach() for k, v in losses.items()}, [p.grad for p in model.parameters() if p.grad is not None]


def test_one_training_step_is_bit_identical():
    det_mode = torch.are_deterministic_algorithms_enabled()
    cudnn = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark)
    torch.use_deterministic_algorithms(True, warn_only=True)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    vision_b200.install()
    try:
        import warnings

        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = _train_step(fused_matching=False)
            got = _train_step(fused_matching=True)
    finally:
        vision_b200.uninstall()
        torch.use_deterministic_algorithms(det_mode)
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = cudnn
    assert want[0].keys() == got[0].keys()
    for k in want[0]:
        assert torch.equal(want[0][k], got[0][k]), k
        assert math.isfinite(want[0][k].item())
    assert len(want[1]) == len(got[1])
    for a, b in zip(want[1], got[1]):
        assert torch.equal(a, b)
