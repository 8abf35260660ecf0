"""GPU suite: RetinaNet's fused head losses against torchvision's own compute_loss bodies on the same seeded inputs, with
matches from det_utils.Matcher(0.5, 0.4, True).  Losses are held to 1e-5 of the reference body run in fp64 (every summand is
>= 0, so nothing cancels); gradients to twice the fp32 reference's own error against that fp64 run, with the rows the
reference leaves at zero exactly zero."""
import copy

import pytest
import torch

tv = pytest.importorskip("torchvision")
from torchvision.models.detection import _utils as det_utils, retinanet  # noqa: E402
from torchvision.ops import boxes as box_ops  # noqa: E402

import vision_b200  # noqa: E402
from vision_b200 import detection as det  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _launches():
    vision_b200._lib.load_ops()
    return torch.ops.vision_b200._launch_count()


def _case(B, C, A, Ms, seed, ignored=(), negative_labels=False, offset=False):
    """B images of A anchors (one shared anchor tensor, as RetinaNet's anchor generator gives each image an equal one), gt
    boxes jittered from random anchors so that a share of anchors match, labels in [0, C) (or [-C, C)), matches from the
    real Matcher; images listed in `ignored` get every anchor ignored (-2).  With `offset` the logits start 4 bytes past an
    allocation, so no image's rows are 16-byte aligned as the gradient's are."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    xy = torch.rand(A, 2, generator=gen, device=DEV) * 480
    anchors = torch.cat([xy, xy + torch.rand(A, 2, generator=gen, device=DEV) * 60 + 8], 1)
    matcher = det_utils.Matcher(0.5, 0.4, True)
    targets, matched = [], []
    for i, M in enumerate(Ms):
        if M:
            pick = torch.randint(0, A, (M,), generator=gen, device=DEV)
            gt = anchors[pick] + (torch.rand(M, 4, generator=gen, device=DEV) - 0.5) * 4
            low = -C if negative_labels else 0
            labels = torch.randint(low, C, (M,), generator=gen, device=DEV)
            m = matcher(box_ops.box_iou(gt, anchors))
        else:
            gt = torch.zeros(0, 4, device=DEV)
            labels = torch.zeros(0, dtype=torch.int64, device=DEV)
            m = torch.full((A,), -1, dtype=torch.int64, device=DEV)
        if i in ignored:
            m = torch.full((A,), -2, dtype=torch.int64, device=DEV)
        targets.append({"boxes": gt, "labels": labels})
        matched.append(m)
    n = B * A * C
    flat = torch.randn(n + (1 if offset else 0), generator=gen, device=DEV) * 2 - 3
    logits = (flat[1:] if offset else flat).view(B, A, C)
    regression = torch.randn(B, A, 4, generator=gen, device=DEV) * 0.5
    return targets, matched, logits, regression, [anchors] * B


def _to64(targets, anchors):
    return ([{"boxes": t["boxes"].double(), "labels": t["labels"]} for t in targets], [a.double() for a in anchors])


def _cls_run(head, targets, matched, logits, fused):
    x = logits.detach().requires_grad_(True)        # not a clone: a misaligned view stays misaligned
    before = _launches()
    if fused:
        vision_b200.install()
    try:
        loss = head.compute_loss(targets, {"cls_logits": x}, matched)
        loss.backward()
    finally:
        vision_b200.uninstall()
    torch.cuda.synchronize()
    assert (_launches() > before) == (fused and x.dtype == torch.float32)
    return loss.detach(), x.grad


def _box_run(head, targets, matched, regression, anchors, fused):
    x = regression.detach().clone().requires_grad_(True)
    before = _launches()
    if fused:
        vision_b200.install()
    try:
        loss = head.compute_loss(targets, {"bbox_regression": x}, anchors, matched)
        loss.backward()
    finally:
        vision_b200.uninstall()
    torch.cuda.synchronize()
    assert (_launches() > before) == (fused and x.dtype == torch.float32)
    return loss.detach(), x.grad


def _check_loss(ours, ref64):
    assert ours.dtype == torch.float32 and ours.dim() == 0 and ours.device.type == "cuda"
    assert abs(ours.double().item() - ref64.item()) <= 1e-5 * abs(ref64.item()), (ours.item(), ref64.item())


def _check_grad(ours, ref32, ref64, zero_rows):
    assert ours.dtype == torch.float32 and ours.shape == ref32.shape and ours.is_contiguous()
    err_ours = (ours.double() - ref64).abs().max().item()
    err_ref = (ref32.double() - ref64).abs().max().item()
    assert err_ours <= 2 * err_ref, (err_ours, err_ref)
    assert torch.all(ours[zero_rows] == 0) and torch.all(ref32[zero_rows] == 0)


CASES = [
    # B, C, A, gt per image, images with every anchor ignored, negative labels, misaligned logits
    (1, 1, 100, [3], (), False, False),                     # below one tile
    (1, 91, 100, [300], (), True, False),
    (2, 2, 1000, [7, 0], (), False, False),                 # a background image; A not a multiple of the tile
    (2, 91, 20001, [50, 7], (), True, False),               # A * C odd: the second image's rows start mid 16-byte group
    (2, 91, 20001, [50, 7], (), False, True),               # logits not 16-byte aligned
    (8, 91, 3000, [1, 50, 0, 300, 7, 2, 20, 5], (5,), True, False),
    (8, 2, 777, [4, 0, 9, 300, 1, 3, 0, 2], (1, 6), False, False),
    (70, 2, 60, [3] * 35 + [0] * 35, (69,), False, False),  # more images than one launch's descriptors
]


@pytest.mark.parametrize("B,C,A,Ms,ignored,negative,offset", CASES)
def test_classification_loss_and_gradient(B, C, A, Ms, ignored, negative, offset):
    targets, matched, logits, _, anchors = _case(B, C, A, Ms, seed=B * 1000 + C * 10 + A, ignored=ignored,
                                                 negative_labels=negative, offset=offset)
    head = retinanet.RetinaNetClassificationHead(8, 1, C)
    ref32, g32 = _cls_run(head, targets, matched, logits, fused=False)
    t64, _ = _to64(targets, anchors)
    ref64, g64 = _cls_run(head, t64, matched, logits.double(), fused=False)
    ours, g = _cls_run(head, targets, matched, logits, fused=True)
    _check_loss(ours, ref64)
    ignored_rows = torch.stack(matched) == -2
    _check_grad(g, g32, g64, ignored_rows)


@pytest.mark.parametrize("B,C,A,Ms,ignored,negative,offset", CASES)
@pytest.mark.parametrize("weights", [(1.0, 1.0, 1.0, 1.0), (10.0, 10.0, 5.0, 5.0), (1.3, 0.7, 2.1, 0.9)])
def test_box_loss_and_gradient(B, C, A, Ms, ignored, negative, offset, weights):
    targets, matched, _, regression, anchors = _case(B, C, A, Ms, seed=B * 1000 + C * 10 + A + 1, ignored=ignored)
    head = retinanet.RetinaNetRegressionHead(8, 1)
    head.box_coder = det_utils.BoxCoder(weights)
    ref32, g32 = _box_run(head, targets, matched, regression, anchors, fused=False)
    t64, a64 = _to64(targets, anchors)
    ref64, g64 = _box_run(head, t64, matched, regression.double(), a64, fused=False)
    ours, g = _box_run(head, targets, matched, regression, anchors, fused=True)
    _check_loss(ours, ref64)
    background_rows = torch.stack(matched) < 0
    _check_grad(g, g32, g64, background_rows)


def test_exact_ties_get_a_zero_gradient():
    """Foreground rows set to the reference's own encode_single targets: |pred - target| is 0 and sign(0) is 0 in both."""
    targets, matched, _, regression, anchors = _case(2, 2, 2000, [30, 12], seed=7)
    head = retinanet.RetinaNetRegressionHead(8, 1)
    head.box_coder = det_utils.BoxCoder((1.3, 0.7, 2.1, 0.9))
    tied = torch.zeros(2, 2000, dtype=torch.bool, device=DEV)
    for i in range(2):
        fg = torch.where(matched[i] >= 0)[0]
        assert fg.numel() > 4
        pick = fg[::2]
        regression[i, pick] = head.box_coder.encode_single(targets[i]["boxes"][matched[i][pick]], anchors[i][pick])
        tied[i, pick] = True
    _, g32 = _box_run(head, targets, matched, regression, anchors, fused=False)
    _, g = _box_run(head, targets, matched, regression, anchors, fused=True)
    assert torch.all(g32[tied] == 0) and torch.all(g[tied] == 0)
    assert torch.all(g[~tied & (torch.stack(matched) >= 0)] != 0)


@pytest.mark.parametrize("value", [float("inf"), float("-inf"), float("nan"), 88.0, -88.0, 0.0, -0.0])
@pytest.mark.parametrize("positive", [False, True])
def test_non_finite_logits_follow_the_reference(value, positive):
    """One logit set to `value` on a foreground anchor, at its target class (t = 1) or another class (t = 0): the loss is
    finite exactly when the reference's is, and the gradient is NaN exactly where the reference's is."""
    targets, matched, logits, _, _ = _case(1, 3, 300, [6], seed=11)
    fg = torch.where(matched[0] >= 0)[0]
    a = int(fg[0])
    k = int(targets[0]["labels"][matched[0][a]]) % 3
    logits[0, a, k if positive else (k + 1) % 3] = value
    head = retinanet.RetinaNetClassificationHead(8, 1, 3)
    ref, gr = _cls_run(head, targets, matched, logits, fused=False)
    ours, g = _cls_run(head, targets, matched, logits, fused=True)
    assert bool(torch.isfinite(ours)) == bool(torch.isfinite(ref))
    assert torch.equal(torch.isnan(g), torch.isnan(gr))


def test_two_calls_are_bit_identical():
    targets, matched, logits, regression, anchors = _case(8, 91, 3000, [1, 50, 0, 300, 7, 2, 20, 5], seed=3, ignored=(5,))
    cls_head, box_head = retinanet.RetinaNetClassificationHead(8, 1, 91), retinanet.RetinaNetRegressionHead(8, 1)
    a = _cls_run(cls_head, targets, matched, logits, fused=True)
    b = _cls_run(cls_head, targets, matched, logits, fused=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    a = _box_run(box_head, targets, matched, regression, anchors, fused=True)
    b = _box_run(box_head, targets, matched, regression, anchors, fused=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_out_of_range_indices_give_a_nan_loss():
    """The reference raises a device-side assert on these, so only the fused ops run: a label outside [-C, C) or a match
    index past the image's gt makes that image's loss NaN."""
    C = 5
    targets, matched, logits, regression, anchors = _case(2, C, 500, [6, 4], seed=5)
    labels = [t["labels"] for t in targets]
    for bad in (C, -C - 1):
        lb = [labels[0], labels[1].clone()]
        lb[1][matched[1][matched[1] >= 0][0]] = bad
        assert torch.isnan(det.retinanet_cls_loss_op(logits, matched, lb))
    m = [matched[0], matched[1].clone()]
    m[1][torch.where(m[1] >= 0)[0][0]] = 4
    assert torch.isnan(det.retinanet_cls_loss_op(logits, m, labels))
    boxes = [t["boxes"] for t in targets]
    assert torch.isnan(det.retinanet_box_loss_op(regression, anchors, boxes, m, [1.0, 1.0, 1.0, 1.0]))
    assert torch.isfinite(det.retinanet_box_loss_op(regression, anchors, boxes, matched, [1.0, 1.0, 1.0, 1.0]))
    assert torch.isfinite(det.retinanet_cls_loss_op(logits, matched, labels))


def test_retinanet_loss_step_does_not_sync_the_host():
    """RetinaNet.compute_loss after install(): matching, both head losses and their backward without a host sync."""
    import types

    targets, matched, logits, regression, anchors = _case(4, 91, 3000, [7, 0, 50, 3], seed=17)
    owner = types.SimpleNamespace(proposal_matcher=det_utils.Matcher(0.5, 0.4, True), head=retinanet.RetinaNetHead(8, 1, 91))

    def step():
        x, r = logits.detach().requires_grad_(True), regression.detach().requires_grad_(True)
        losses = retinanet.RetinaNet.compute_loss(owner, targets, {"cls_logits": x, "bbox_regression": r}, anchors)
        (losses["classification"] + losses["bbox_regression"]).backward()
        return x.grad

    vision_b200.install()
    try:
        before = _launches()
        step()                                      # loads the ops and warms autograd outside the checked region
        assert _launches() > before
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            step()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    finally:
        vision_b200.uninstall()


def test_training_step_matches_the_reference_losses():
    """One training step of retinanet_resnet50_fpn with install() against install() without the two head-loss rebinds;
    cuDNN is made deterministic so that the convolutions add no noise of their own (each path is then bit-reproducible).
    Only the head losses differ.  The focal loss sums in another order with other (stable) formulas: its value agrees to
    1e-5 relative and d loss / d cls_logits to 1e-6 of its largest entry (1.7e-7 measured on an H100).  The box loss's
    gradient has the reference's bits, so it must be equal.  Back-propagated through the untrained backbone, whose
    BatchNorm layers in training mode subtract batch means from nearly equal terms, those 1e-7 differences grow about
    10^4-fold (2.6e-3 of the largest entry at worst, in the backbone's BatchNorm biases, measured on an H100).  The
    parameter gradients are therefore held to 2e-2 of each one's largest entry: above that rounding growth, and far below
    what a wrong scale, a dropped image or a misplaced row gives (a change of order 1)."""
    from torchvision.models.detection import retinanet_resnet50_fpn

    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    torch.manual_seed(0)
    model = retinanet_resnet50_fpn(weights=None, weights_backbone=None).to(DEV).train()
    gen = torch.Generator(device=DEV).manual_seed(1)
    images = [torch.rand(3, 480, 640, generator=gen, device=DEV) for _ in range(2)]
    targets = []
    for m in (5, 3):
        xy = torch.rand(m, 2, generator=gen, device=DEV) * 400
        targets.append({"boxes": torch.cat([xy, xy + 40 + torch.rand(m, 2, generator=gen, device=DEV) * 150], 1),
                        "labels": torch.randint(1, 91, (m,), generator=gen, device=DEV)})
    state = copy.deepcopy(model.state_dict())
    head_outputs = {}
    head_forward = model.head.forward

    def keep_head_outputs(x):
        out = head_forward(x)
        for k, v in out.items():
            v.retain_grad()
            head_outputs[k] = v
        return out

    model.head.forward = keep_head_outputs

    def step(rebind_losses):
        model.load_state_dict(state)
        model.zero_grad(set_to_none=True)
        vision_b200.install()
        try:
            if not rebind_losses:
                from vision_b200 import _install

                for (cls, name), orig in _install._state["losses"].items():
                    setattr(cls, name, orig)
            losses = model(images, targets)
            sum(losses.values()).backward()
        finally:
            vision_b200.uninstall()
        return ({k: v.detach() for k, v in losses.items()}, {k: v.grad.clone() for k, v in head_outputs.items()},
                {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None})

    try:
        fused_losses, fused_heads, fused_grads = step(True)
        ref_losses, ref_heads, ref_grads = step(False)
    finally:
        torch.backends.cudnn.deterministic = False
    assert fused_losses.keys() == ref_losses.keys() == {"classification", "bbox_regression"}
    for k in ref_losses:
        assert abs(fused_losses[k].item() - ref_losses[k].item()) <= 1e-5 * abs(ref_losses[k].item()), k
    g = ref_heads["cls_logits"]
    assert (fused_heads["cls_logits"] - g).abs().max().item() <= 1e-6 * g.abs().max().item()
    assert torch.equal(fused_heads["bbox_regression"], ref_heads["bbox_regression"])
    assert fused_grads.keys() == ref_grads.keys()
    for n, g in ref_grads.items():
        assert (fused_grads[n] - g).abs().max().item() <= 2e-2 * g.abs().max().item(), n
