"""GPU suite: FCOS's fused head losses against torchvision's own FCOSHead.compute_loss body on the same seeded inputs, with
matches from the fused FCOS matcher (bit-identical to the reference's).  Losses are held to 1e-5 of the reference body run in
fp64 (every summand -- focal, GIoU, BCE -- is >= 0, so nothing cancels); gradients to twice the fp32 reference's own error
against that fp64 run, with the box and centre-ness rows the reference leaves at zero exactly zero."""
import copy
import math
import types

import pytest
import torch

tv = pytest.importorskip("torchvision")
from torchvision.models.detection import _utils as det_utils, fcos  # noqa: E402

import vision_b200  # noqa: E402
from vision_b200 import detection as det  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
STRIDES = (8, 16, 32, 64, 128)


def _launches():
    vision_b200._lib.load_ops()
    return torch.ops.vision_b200._launch_count()


def _anchors(H, W):
    """FCOS's anchors for an H x W batch: per level of stride s a square of side s around each (x·s, y·s), levels in order."""
    rows, levels = [], []
    for s in STRIDES:
        h, w = -(-H // s), -(-W // s)
        y, x = torch.meshgrid(torch.arange(h, device=DEV) * s, torch.arange(w, device=DEV) * s, indexing="ij")
        c = torch.stack([x.reshape(-1), y.reshape(-1)], 1).float()
        rows.append(torch.cat([c - s / 2, c + s / 2], 1))
        levels.append(h * w)
    return torch.cat(rows), levels


def _case(B, C, H, W, Ms, seed, negative_labels=False, offset=False, minus_two=False, normalize=True):
    """B images of H x W (one anchor tensor per image, as FCOS's generator gives), integer gt boxes inside the image, labels
    in [0, C) (or [-C, C)), matches from the fused FCOS matcher; `minus_two` turns a share of the matches into -2; with
    `offset` the logits start 4 bytes past an allocation.  Regression codes are positive distances, per anchor size when
    normalising."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    anchors, levels = _anchors(H, W)
    A = anchors.shape[0]
    targets = []
    for M in Ms:
        lo = torch.randint(0, max(H, W) // 2, (M, 2), generator=gen, device=DEV)
        size = torch.randint(8, max(H, W) // 2, (M, 2), generator=gen, device=DEV)
        boxes = torch.cat([lo, lo + size], 1).float()
        labels = torch.randint(-C if negative_labels else 0, C, (M,), generator=gen, device=DEV)
        targets.append({"boxes": boxes, "labels": labels})
    matched = det.fcos_match_op([t["boxes"] for t in targets], [anchors] * B, 1.5, levels)
    if minus_two:
        for m in matched:
            m[torch.rand(A, generator=gen, device=DEV) < 0.3] = -2
    flat = torch.randn(B * A * C + (1 if offset else 0), generator=gen, device=DEV) * 2 - 3
    logits = (flat[1:] if offset else flat).view(B, A, C)
    regression = torch.rand(B, A, 4, generator=gen, device=DEV) * 3 + 0.05
    if not normalize:
        regression = regression * (anchors[:, 2] - anchors[:, 0])[None, :, None]
    ctrness = torch.randn(B, A, 1, generator=gen, device=DEV)
    outputs = {"cls_logits": logits, "bbox_regression": regression, "bbox_ctrness": ctrness}
    return targets, outputs, [anchors] * B, matched


def _head(C, normalize=True):
    head = fcos.FCOSHead(32, 1, C, num_convs=1)
    head.box_coder = det_utils.BoxLinearCoder(normalize)
    return head


def _run(head, targets, outputs, anchors, matched, fused, dtype=torch.float32):
    """compute_loss and the backward of the three losses' sum: the losses and d/d each head output."""
    xs = {k: (v.detach() if dtype == torch.float32 else v.detach().to(dtype)).requires_grad_(True) for k, v in outputs.items()}
    if dtype != torch.float32:
        targets = [{"boxes": t["boxes"].to(dtype), "labels": t["labels"]} for t in targets]
        anchors = [a.to(dtype) for a in anchors]
    before = _launches()
    if fused:
        vision_b200.install()
    try:
        losses = head.compute_loss(targets, xs, anchors, matched)
        sum(losses.values()).backward()
    finally:
        vision_b200.uninstall()
    torch.cuda.synchronize()
    assert (_launches() > before) == (fused and dtype == torch.float32)
    return {k: v.detach() for k, v in losses.items()}, {k: v.grad for k, v in xs.items()}


def _foreground(targets, matched):
    """The reference's foreground mask (fcos.py:64-85)."""
    rows = []
    for t, m in zip(targets, matched):
        cls = t["labels"][m.clip(min=0)] if len(t["labels"]) else torch.zeros_like(m)
        rows.append((cls >= 0) & (m >= 0))
    return torch.stack(rows)


def _check_loss(ours, ref64):
    assert ours.dtype == torch.float32 and ours.dim() == 0 and ours.device.type == "cuda"
    assert abs(ours.double().item() - ref64.item()) <= 1e-5 * abs(ref64.item()), (ours.item(), ref64.item())


def _check_grad(ours, ref32, ref64, zero_rows=None):
    assert ours.dtype == torch.float32 and ours.shape == ref32.shape and ours.is_contiguous()
    err_ours = (ours.double() - ref64).abs().max().item()
    err_ref = (ref32.double() - ref64).abs().max().item()
    assert err_ours <= 2 * err_ref, (err_ours, err_ref)
    if zero_rows is not None:
        assert torch.all(ours[zero_rows] == 0) and torch.all(ref32[zero_rows] == 0)


CASES = [
    # B, C, H, W, gt per image, negative labels, misaligned logits, -2 matches, normalize_by_size
    (1, 3, 64, 64, [3], False, False, False, True),                 # below one tile (86 anchors)
    (2, 1, 200, 264, [5, 2], False, False, False, True),            # C = 1
    (2, 91, 200, 264, [7, 50], True, False, False, True),           # A odd: the second image's rows start mid 16-byte group
    (2, 91, 200, 264, [7, 50], False, True, False, True),           # logits not 16-byte aligned
    (3, 5, 400, 520, [4, 0, 6], False, False, True, True),          # an image without gt; -2 matches
    (2, 5, 200, 264, [0, 0], False, False, False, True),            # no foreground in the batch: n = 0
    (2, 7, 200, 264, [9, 3], True, False, True, False),             # normalize_by_size=False
    (70, 2, 64, 64, [2] * 35 + [0] * 35, False, False, False, True),  # more images than one launch's descriptors
]


@pytest.mark.parametrize("B,C,H,W,Ms,negative,offset,minus_two,normalize", CASES)
def test_losses_and_gradients(B, C, H, W, Ms, negative, offset, minus_two, normalize):
    targets, outputs, anchors, matched = _case(B, C, H, W, Ms, seed=B * 1000 + C * 10 + H, negative_labels=negative, offset=offset,
                                               minus_two=minus_two, normalize=normalize)
    head = _head(C, normalize)
    ref32, g32 = _run(head, targets, outputs, anchors, matched, fused=False)
    ref64, g64 = _run(head, targets, outputs, anchors, matched, fused=False, dtype=torch.float64)
    ours, g = _run(head, targets, outputs, anchors, matched, fused=True)
    background = ~_foreground(targets, matched)
    if not sum(Ms):
        assert ours["bbox_regression"].item() == 0 and ours["bbox_ctrness"].item() == 0
    for k in ("classification", "bbox_regression", "bbox_ctrness"):
        _check_loss(ours[k], ref64[k])
    _check_grad(g["cls_logits"], g32["cls_logits"], g64["cls_logits"])
    _check_grad(g["bbox_regression"], g32["bbox_regression"], g64["bbox_regression"], background)
    _check_grad(g["bbox_ctrness"], g32["bbox_ctrness"], g64["bbox_ctrness"], background)


def test_ties_take_half_the_gradient():
    """Foreground predictions decoded exactly onto their gt's left and top edges (power-of-two anchor sizes, integer boxes,
    exact codes) and 1/4 of the anchor size inside the right and bottom ones: torch.max / torch.min give each side of those
    ties half the gradient.  The fused gradient matches the fp32 reference's within 1e-6 of each row's largest entry; a
    full or a zero share would be off by order 1."""
    targets, outputs, anchors, matched = _case(2, 3, 200, 264, [6, 4], seed=21)
    regression = outputs["bbox_regression"]
    tied = torch.zeros(regression.shape[:2], dtype=torch.bool, device=DEV)
    a = anchors[0]
    cx, cy, s = (a[:, 0] + a[:, 2]) / 2, (a[:, 1] + a[:, 3]) / 2, a[:, 2] - a[:, 0]
    for i in range(2):
        fg = torch.where(matched[i] >= 0)[0]
        assert fg.numel() > 4
        g = targets[i]["boxes"][matched[i][fg]]
        q = s[fg] / 4
        codes = torch.stack([cx[fg] - g[:, 0], cy[fg] - g[:, 1], g[:, 2] - q - cx[fg], g[:, 3] - q - cy[fg]], 1) / s[fg, None]
        regression[i, fg] = codes
        tied[i, fg] = True
    head = _head(3)
    _, g32 = _run(head, targets, outputs, anchors, matched, fused=False)
    _, g = _run(head, targets, outputs, anchors, matched, fused=True)
    ref, ours = g32["bbox_regression"][tied], g["bbox_regression"][tied]
    scale = ref.abs().amax(dim=1, keepdim=True)
    assert torch.all(scale > 0)
    assert torch.all((ours - ref).abs() <= 1e-6 * scale), ((ours - ref).abs() / scale).max().item()


def test_out_of_range_indices_give_a_nan_loss():
    """The reference raises a device-side assert on these, so only the fused ops run: a match index past the image's gt
    makes all three losses NaN, a label >= C the classification loss (the box call reads no class)."""
    C = 5
    targets, outputs, anchors, matched = _case(2, C, 200, 264, [6, 4], seed=5)
    labels = [t["labels"] for t in targets]
    boxes = [t["boxes"] for t in targets]
    args = (outputs["bbox_regression"], outputs["bbox_ctrness"], anchors, boxes)
    assert torch.isfinite(det.fcos_cls_loss_op(outputs["cls_logits"], matched, labels))
    assert all(torch.isfinite(x) for x in det.fcos_box_loss_op(*args, labels, matched, True))
    m = [matched[0], matched[1].clone()]
    m[1][torch.where(m[1] >= 0)[0][0]] = 4
    assert torch.isnan(det.fcos_cls_loss_op(outputs["cls_logits"], m, labels))
    assert all(torch.isnan(x) for x in det.fcos_box_loss_op(*args, labels, m, True))
    lb = [labels[0], labels[1].clone()]
    lb[1][matched[1][matched[1] >= 0][0]] = C
    assert torch.isnan(det.fcos_cls_loss_op(outputs["cls_logits"], matched, lb))


def test_two_calls_are_bit_identical():
    targets, outputs, anchors, matched = _case(8, 91, 200, 264, [1, 50, 0, 30, 7, 2, 20, 5], seed=3, minus_two=True)
    head = _head(91)
    a = _run(head, targets, outputs, anchors, matched, fused=True)
    b = _run(head, targets, outputs, anchors, matched, fused=True)
    for k in a[0]:
        assert torch.equal(a[0][k], b[0][k]), k
    for k in a[1]:
        assert torch.equal(a[1][k], b[1][k]), k


def _owner(C):
    return types.SimpleNamespace(center_sampling_radius=1.5, head=_head(C))


def test_fcos_loss_step_does_not_sync_the_host():
    """FCOS.compute_loss after install(): the fused matcher, the three head losses and their backward without a host sync."""
    targets, outputs, anchors, _ = _case(4, 91, 200, 264, [7, 0, 50, 3], seed=17)
    levels = _anchors(200, 264)[1]
    owner = _owner(91)

    def step():
        xs = {k: v.detach().requires_grad_(True) for k, v in outputs.items()}
        losses = fcos.FCOS.compute_loss(owner, targets, xs, anchors, levels)
        sum(losses.values()).backward()

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


def test_launch_count_does_not_grow_with_the_batch():
    counts = []
    for B in (1, 8):
        targets, outputs, anchors, matched = _case(B, 91, 200, 264, [5] * B, seed=B)
        head = _head(91)
        xs = {k: v.detach().requires_grad_(True) for k, v in outputs.items()}
        vision_b200.install()
        try:
            torch.cuda.synchronize()
            before = _launches()
            losses = head.compute_loss(targets, xs, anchors, matched)
            sum(losses.values()).backward()
            counts.append(_launches() - before)
        finally:
            vision_b200.uninstall()
    assert counts[0] == counts[1] == 6, counts      # per loss call: forward + finalize, then one backward


def test_training_step_matches_the_reference_losses():
    """One training step of fcos_resnet50_fpn with install() (fused matcher and head loss) against install() with the
    FCOSHead rebinding restored; cuDNN is made deterministic so that the convolutions add no noise of their own.  Only the
    head loss differs.  Its values agree to 1e-5 relative and d loss / d cls_logits to 1e-6 of its largest entry (the
    focal terms of test_gpu_retinanet_loss.py).  The box and centre-ness gradients are computed in fp64 from the fp32
    forward's decisions where the reference chains fp32 autograd ops: measured on an H100, they differ from the reference's
    by 1.5e-6 (box) and 9.5e-8 (centre-ness) of their largest entry, and are held to 1e-5 and 1e-6.  Through the untrained
    backbone's BatchNorm those differences grow about 10^4-fold, so the parameter gradients are held to 2e-2 of each one's
    largest entry, as in test_gpu_retinanet_loss.py."""
    from torchvision.models.detection import fcos_resnet50_fpn

    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    torch.manual_seed(0)
    model = fcos_resnet50_fpn(weights=None, weights_backbone=None).to(DEV).train()
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

    def step(fused_head_loss):
        model.load_state_dict(state)
        model.zero_grad(set_to_none=True)
        vision_b200.install()
        try:
            if not fused_head_loss:
                from vision_b200 import _install

                for (cls, name), orig in _install._state["fcos_losses"].items():
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
    assert fused_losses.keys() == ref_losses.keys() == {"classification", "bbox_regression", "bbox_ctrness"}
    for k in ref_losses:
        assert math.isfinite(ref_losses[k].item())
        assert abs(fused_losses[k].item() - ref_losses[k].item()) <= 1e-5 * abs(ref_losses[k].item()), k
    rel = {k: ((fused_heads[k] - g).abs().max() / g.abs().max()).item() for k, g in ref_heads.items()}
    print(f"head-output gradient differences over their largest entries: {rel}")
    assert rel["cls_logits"] <= 1e-6
    assert rel["bbox_regression"] <= 1e-5 and rel["bbox_ctrness"] <= 1e-6
    assert fused_grads.keys() == ref_grads.keys()
    for n, g in ref_grads.items():
        assert (fused_grads[n] - g).abs().max().item() <= 2e-2 * g.abs().max().item(), n
