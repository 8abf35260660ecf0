"""GPU suite: the fused training-target assignment against the reference on the same GPU, bit for bit.  Op-level cases
compare vision_b200::match_boxes with Matcher(high, low, allow)(box_iou(gt, boxes)); method-level cases compare the three
rebound methods with the same methods uninstalled; one training step of three detection models compares full install()
with install() minus the three matching rebinds, so both sides run the same roi_align and NMS kernels."""
import math

import numpy as np
import pytest
import torch

tv = pytest.importorskip("torchvision")
from torchvision.models.detection import _utils as det_utils, retinanet, roi_heads, rpn  # noqa: E402
from torchvision.ops import boxes as box_ops  # noqa: E402

import vision_b200  # noqa: E402
from vision_b200 import detection as det  # noqa: E402

pytestmark = pytest.mark.gpu

RPN, RETINANET, ROI_HEADS = (0.7, 0.3, True), (0.5, 0.4, True), (0.5, 0.5, False)
SETTINGS = {"rpn": RPN, "retinanet": RETINANET, "roi_heads": ROI_HEADS}
RPN_ANCHORS = 217_413          # RPN anchors of an 800 x 1088 input (5 FPN levels, 3 aspect ratios)


def _boxes(n, gen, w=1088.0, h=800.0):
    c = torch.rand(n, 2, generator=gen) * torch.tensor([w, h])
    s = torch.rand(n, 2, generator=gen) * 300 + 4
    return torch.cat([c - s / 2, c + s / 2], 1)


def _problem(M, N, seed=0):
    """Random gt and predictions, a quarter of the predictions jittered copies of gt boxes so every threshold band is hit."""
    gen = torch.Generator().manual_seed(seed)
    gt = _boxes(M, gen)
    pred = _boxes(N, gen)
    k = N // 4
    if k and M:
        src = gt[torch.randint(0, M, (k,), generator=gen)]
        pred[:k] = src + torch.randn(k, 4, generator=gen) * (src[:, 2:] - src[:, :2]).repeat(1, 2) * 0.15
    return gt.cuda(), pred.cuda()


def _reference(gt, pred, setting):
    return det_utils.Matcher(*setting)(box_ops.box_iou(gt, pred))


def _fused(gts, preds, setting, mode=det.MATCH_RAW, labels=None):
    out0, out1 = det.match_boxes_op(gts, preds, labels, det_utils.Matcher(*setting), mode)
    return out0 if mode == det.MATCH_RAW else (out0, out1)


def _same(got, want):
    if isinstance(want, (list, tuple)):
        assert len(got) == len(want)
        for g, w in zip(got, want):
            _same(g, w)
        return
    assert got.dtype == want.dtype and got.shape == want.shape and got.stride() == want.stride() and got.device == want.device
    assert torch.equal(got, want)


@pytest.mark.parametrize("setting", SETTINGS)
@pytest.mark.parametrize("N", [1, 1000, RPN_ANCHORS])
@pytest.mark.parametrize("M", [1, 3, 50, 300])
def test_matches_equal_the_reference(M, N, setting):
    gt, pred = _problem(M, N, seed=M * 7 + N)
    _same(_fused([gt], [pred], SETTINGS[setting])[0], _reference(gt, pred, SETTINGS[setting]))


@pytest.mark.parametrize("setting", SETTINGS)
def test_images_of_different_sizes_in_one_call(setting):
    probs = [_problem(M, N, seed=i) for i, (M, N) in enumerate([(7, 5000), (1, 30), (300, 2200), (50, RPN_ANCHORS), (2, 1)])]
    got = _fused([g for g, _ in probs], [p for _, p in probs], SETTINGS[setting])
    _same(got, [_reference(g, p, SETTINGS[setting]) for g, p in probs])


def _special_problem():
    """Duplicate gt boxes (the lowest index wins), duplicate predictions (ties in a gt's max), a gt far from every
    prediction (its max is 0, so every prediction with IoU 0 to it is a low-quality match), NaN and -0.0 coordinates and
    inverted (negative-area) predictions."""
    gt, pred = _problem(12, 3000, seed=5)
    gt = gt.clone()
    pred = pred.clone()
    gt[3] = gt[1]
    gt[7] = gt[1]
    gt[10] = torch.tensor([5000.0, 5000.0, 5100.0, 5100.0])
    pred[100:110] = pred[5]
    pred[200:210] = gt[4]
    pred[300, 0] = float("nan")
    pred[301, 3] = float("nan")
    gt[11, 2] = float("nan")
    pred[400:420, 0] = -0.0
    pred[400:420, 2] = pred[400:420, 2].abs() + 1
    gt[0, 1] = -0.0
    pred[500:600] = pred[500:600][:, [2, 3, 0, 1]]
    pred[600:650, 2] = pred[600:650, 0] - 5
    return gt, pred


@pytest.mark.parametrize("setting", SETTINGS)
def test_duplicates_disjoint_gt_nan_signed_zero_and_inverted_boxes(setting):
    gt, pred = _special_problem()
    _same(_fused([gt], [pred], SETTINGS[setting])[0], _reference(gt, pred, SETTINGS[setting]))


def test_ious_at_the_float_thresholds_and_one_ulp_either_side():
    gt, pred = _problem(20, 4000, seed=11)
    iou = box_ops.box_iou(gt, pred)
    vals = iou.max(0).values
    picks = vals[(vals > 0.05) & (vals < 0.95)][:8].cpu().numpy().astype(np.float32)
    for v in picks:
        down, up = np.nextafter(v, np.float32(0)), np.nextafter(v, np.float32(1))
        # float(v) + 1e-12 is not an fp32 value but rounds to v, as torch rounds a Python float compared with an fp32 tensor
        for low, high in ((float(v), float(up)), (float(down), float(v)), (float(v), float(v)), (float(v) + 1e-12, float(up) + 1e-12)):
            for allow in (False, True):
                setting = (high, low, allow)
                _same(_fused([gt], [pred], setting)[0], _reference(gt, pred, setting))


@pytest.mark.parametrize("gt_dtype,pred_dtype", [(torch.float32, torch.float16), (torch.float32, torch.bfloat16),
                                                 (torch.float16, torch.float16), (torch.bfloat16, torch.bfloat16),
                                                 (torch.float16, torch.bfloat16), (torch.bfloat16, torch.float32),
                                                 (torch.float64, torch.float64)])
@pytest.mark.parametrize("setting", SETTINGS)
def test_dtypes(gt_dtype, pred_dtype, setting):
    gt, pred = _special_problem()
    gt, pred = gt.to(gt_dtype), pred.to(pred_dtype)
    _same(_fused([gt], [pred], SETTINGS[setting])[0], _reference(gt, pred, SETTINGS[setting]))


# ---- the three methods --------------------------------------------------------------------------------------------------

def _owners():
    import types

    head = types.SimpleNamespace(compute_loss=lambda targets, outputs, anchors, matched: matched)
    return (types.SimpleNamespace(box_similarity=box_ops.box_iou, proposal_matcher=det_utils.Matcher(*RPN)),
            types.SimpleNamespace(proposal_matcher=det_utils.Matcher(*ROI_HEADS)),
            types.SimpleNamespace(proposal_matcher=det_utils.Matcher(*RETINANET), head=head))


def _call_all(gts, preds, labels):
    r, h, n = _owners()
    return (rpn.RegionProposalNetwork.assign_targets_to_anchors(r, preds, [{"boxes": g} for g in gts]),
            roi_heads.RoIHeads.assign_targets_to_proposals(h, preds, gts, labels),
            retinanet.RetinaNet.compute_loss(n, [{"boxes": g} for g in gts], {}, preds))


def _installed(fn):
    vision_b200.install()
    try:
        before = vision_b200.launch_count()
        out = fn()
        torch.cuda.synchronize()
        return out, vision_b200.launch_count() - before
    finally:
        vision_b200.uninstall()


def _batch(B, seed=0, background=(), gt_dtype=torch.float32, pred_dtype=torch.float32):
    gts, preds, labels = [], [], []
    for i in range(B):
        g, p = _problem(0 if i in background else 3 + 5 * i, 2000 + 17 * i, seed=seed + i)
        gts.append(g.to(gt_dtype))
        preds.append(p.to(pred_dtype))
        labels.append(torch.randint(1, 91, (g.shape[0],), device="cuda"))
    return gts, preds, labels


@pytest.mark.parametrize("case", ["plain", "background", "all_background", "fp16_anchors", "fp64"])
def test_methods_equal_the_uninstalled_ones(case):
    kw = {"plain": {}, "background": {"background": (1, 3)}, "all_background": {"background": (0, 1, 2, 3)},
          "fp16_anchors": {"pred_dtype": torch.float16}, "fp64": {"gt_dtype": torch.float64, "pred_dtype": torch.float64}}[case]
    gts, preds, labels = _batch(4, **kw)
    if case == "background":
        gts[1] = torch.zeros(0, 4, device="cuda")          # a [0, 4] and a [0] gt: both are background images
        gts[3] = torch.zeros(0, device="cuda")
    want = _call_all(gts, preds, labels)
    got, _ = _installed(lambda: _call_all(gts, preds, labels))
    _same(got, want)


def test_no_predictions_raise_the_reference_error():
    gts, preds, labels = _batch(2)
    preds[1] = preds[1][:0]
    for call in range(3):
        with pytest.raises(ValueError, match="No proposal boxes available for one of the images during training"):
            _call_all_one(call, gts, preds, labels)
        vision_b200.install()
        try:
            with pytest.raises(ValueError, match="No proposal boxes available for one of the images during training"):
                _call_all_one(call, gts, preds, labels)
        finally:
            vision_b200.uninstall()


def _call_all_one(which, gts, preds, labels):
    r, h, n = _owners()
    if which == 0:
        return rpn.RegionProposalNetwork.assign_targets_to_anchors(r, preds, [{"boxes": g} for g in gts])
    if which == 1:
        return roi_heads.RoIHeads.assign_targets_to_proposals(h, preds, gts, labels)
    return retinanet.RetinaNet.compute_loss(n, [{"boxes": g} for g in gts], {}, preds)


def test_rpn_and_retinanet_matching_do_not_sync_the_host():
    gts, preds, labels = _batch(4, background=(2,))
    r, _, n = _owners()
    _installed(lambda: None)                     # loads the ops outside the checked region
    vision_b200.install()
    try:
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            rpn.RegionProposalNetwork.assign_targets_to_anchors(r, preds, [{"boxes": g} for g in gts])
            retinanet.RetinaNet.compute_loss(n, [{"boxes": g} for g in gts], {}, preds)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    finally:
        vision_b200.uninstall()


def test_launch_count_does_not_grow_with_the_batch():
    counts = []
    for B in (1, 8):
        gts, preds, labels = _batch(B)
        _, launches = _installed(lambda: _call_all(gts, preds, labels))
        counts.append(launches)
    # RPN and RetinaNet: the gt maxima and the matches; RoIHeads: the matches
    assert counts[0] == counts[1] == 5


# ---- one training step ----------------------------------------------------------------------------------------------------

def _train_step(builder, fused_matching: bool):
    from vision_b200 import _install

    torch.manual_seed(0)
    model = builder(weights=None, weights_backbone=None, num_classes=5, min_size=320, max_size=448).cuda().train()
    gen = torch.Generator().manual_seed(1)
    images = [torch.rand(3, 300 + 40 * i, 420 - 30 * i, generator=gen).cuda() for i in range(2)]
    targets = []
    for i, img in enumerate(images):
        h, w = img.shape[1:]
        xy = torch.rand(3 + i, 2, generator=gen) * torch.tensor([w * 0.6, h * 0.6])
        wh = torch.rand(3 + i, 2, generator=gen) * torch.tensor([w * 0.35, h * 0.35]) + 8
        t = {"boxes": torch.cat([xy, xy + wh], 1).cuda(), "labels": torch.randint(1, 5, (3 + i,), generator=gen).cuda()}
        if builder is tv.models.detection.maskrcnn_resnet50_fpn:
            t["masks"] = (torch.rand(3 + i, h, w, generator=gen) > 0.5).to(torch.uint8).cuda()
        targets.append(t)
    saved = {}
    if not fused_matching:
        for (cls, name), orig in _install._state["matching"].items():
            saved[(cls, name)] = getattr(cls, name)
            setattr(cls, name, orig)
    try:
        torch.manual_seed(2)
        losses = model(images, targets)
        sum(losses.values()).backward()
    finally:
        for (cls, name), fn in saved.items():
            setattr(cls, name, fn)
    torch.cuda.synchronize()
    return {k: v.detach() for k, v in losses.items()}, [p.grad for p in model.parameters() if p.grad is not None]


@pytest.mark.parametrize("name", ["fasterrcnn_resnet50_fpn", "maskrcnn_resnet50_fpn", "retinanet_resnet50_fpn"])
def test_one_training_step_is_bit_identical(name):
    builder = getattr(tv.models.detection, name)
    det_mode = torch.are_deterministic_algorithms_enabled()
    cudnn = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark)
    torch.use_deterministic_algorithms(True, warn_only=True)
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    vision_b200.install()
    try:
        import warnings

        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            want = _train_step(builder, fused_matching=False)
            got = _train_step(builder, fused_matching=True)
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
