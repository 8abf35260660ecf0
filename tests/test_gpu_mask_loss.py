"""GPU suite: Mask R-CNN's fused mask loss against torchvision's own maskrcnn_loss on seeded inputs.  Targets must have the
bits of the reference CPU roi_align over the masks as fp32; the loss is held to 1e-5 of BCE-with-logits in fp64 against
those targets; the gradient to twice the fp32 reference body's own error against the fp64 gradient, with every plane but
each RoI's label plane exactly zero."""
import copy

import pytest
import torch
import torch.nn.functional as F

tv = pytest.importorskip("torchvision")
from torchvision.models.detection import roi_heads  # noqa: E402
from torchvision.ops import roi_align  # noqa: E402

import vision_b200  # noqa: E402
from vision_b200 import detection as det  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _launches():
    vision_b200._lib.load_ops()
    return torch.ops.vision_b200._launch_count()


def _masks(G, H, W, gen):
    """G blob masks: random ellipses, so that targets take every value in [0, 1]."""
    yy = torch.arange(H, device=DEV, dtype=torch.float32)[:, None]
    xx = torch.arange(W, device=DEV, dtype=torch.float32)[None, :]
    c = torch.rand(G, 4, generator=gen, device=DEV)
    cy, cx = c[:, 0, None, None] * H, c[:, 1, None, None] * W
    ry, rx = 2 + c[:, 2, None, None] * H / 2, 2 + c[:, 3, None, None] * W / 2
    return (((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1).to(torch.uint8)


def _case(name="plain", M=28, C=7, seed=0):
    """(mask_logits, proposals, gt_masks, gt_labels, matched) of one named geometry, every tensor on the GPU."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    sizes = {"sizes": [(40, 56), (63, 31), (17, 90)], "large": [(800, 1088), (640, 704)],
             "many": [(24 + i % 5, 30 + i % 7) for i in range(70)]}.get(name, [(48, 64), (50, 40)])
    positives = {"empty_image": [6, 0, 5]}.get(name, [9] * len(sizes))
    if name == "empty_image":
        sizes = [(48, 64), (30, 30), (50, 40)]
    proposals, masks, labels, matched = [], [], [], []
    for i, ((H, W), P) in enumerate(zip(sizes, positives)):
        G = 3 + (H % 3)
        g = _masks(G, H, W, gen)
        m = torch.randint(0, G, (P,), generator=gen, device=DEV)
        xy = torch.rand(P, 2, generator=gen, device=DEV) * torch.tensor([W, H], device=DEV) * 0.8
        wh = 1 + torch.rand(P, 2, generator=gen, device=DEV) * torch.tensor([W, H], device=DEV) * 0.6
        box = torch.cat([xy, xy + wh], 1)
        if name == "outside" and P:
            box[0] = torch.tensor([-20.0, -10.0, W * 0.5, H * 0.5])               # partly outside, top-left
            box[1] = torch.tensor([W * 0.5, H * 0.5, W + 30.0, H + 12.0])          # partly outside, bottom-right
            box[2] = torch.tensor([W + 5.0, H + 5.0, W + 40.0, H + 33.0])          # wholly outside
            box[3] = torch.tensor([-50.0, -40.0, -3.0, -2.0])                      # wholly outside, negative
        if name == "degenerate" and P:
            box[0] = torch.tensor([10.0, 12.0, 10.0, 30.0])                        # zero width
            box[1] = torch.tensor([20.0, 20.0, 5.0, 8.0])                          # inverted
            box[2] = torch.tensor([7.5, 9.25, 7.5, 9.25])                          # a point
        if name == "one_sample":
            box = torch.cat([xy, xy + torch.rand(P, 2, generator=gen, device=DEV) * (M - 1)], 1)
        if name == "large" and P:
            box[0] = torch.tensor([0.0, 0.0, W - 1.0, H - 1.0])                    # image-sized, > 504 px both ways
            box[1] = torch.tensor([-30.0, 100.0, W + 20.0, 140.0])                 # > 504 px wide
            box[2] = torch.tensor([10.0, -5.0, 60.0, H + 7.0])                     # > 504 px tall
        if name == "bool":
            g = g.bool()
        if name == "noncontiguous":
            g = g.transpose(1, 2).contiguous().transpose(1, 2) if i % 2 == 0 else torch.cat([g, g], 2)[:, :, ::2]
        proposals.append(box.contiguous())
        masks.append(g)
        labels.append(torch.randint(1, C, (G,), generator=gen, device=DEV))
        matched.append(m)
    P = sum(positives)
    logits = torch.randn(P, C, M, M, generator=gen, device=DEV) * 3
    return logits, proposals, masks, labels, matched


def _reference_targets(proposals, masks, matched, M):
    """project_masks_on_boxes with the reference CPU roi_align over the masks as fp32."""
    out = []
    for p, g, m in zip(proposals, masks, matched):
        rois = torch.cat([m.to(p)[:, None], p], 1).cpu()
        out.append(roi_align(g[:, None].float().cpu(), rois, (M, M), 1.0)[:, 0])
    return torch.cat(out, 0)


def _truth64(logits, targets, labels, matched):
    """Loss and d loss / d mask_logits in fp64 against the given targets."""
    lab = torch.cat([l[m] for l, m in zip(labels, matched)]).cpu()
    x = logits.detach().double().cpu().requires_grad_(True)
    idx = torch.arange(lab.shape[0])
    loss = F.binary_cross_entropy_with_logits(x[idx, lab], targets.double())
    loss.backward()
    return loss.item(), x.grad, lab


CASES = ["plain", "outside", "degenerate", "large", "one_sample", "bool", "noncontiguous", "sizes", "empty_image", "many"]


@pytest.mark.parametrize("M", [14, 28, 56])
@pytest.mark.parametrize("name", CASES)
def test_targets_loss_and_gradient(name, M):
    if name in ("large", "many") and M != 28:
        pytest.skip("one output size is enough for the large and many-image geometries")
    logits, proposals, masks, labels, matched = _case(name, M=M)
    x = logits.clone().requires_grad_(True)
    loss, targets = det.maskrcnn_loss_op(x, proposals, masks, labels, matched)
    loss.backward()
    want = _reference_targets(proposals, masks, matched, M)
    assert torch.equal(targets.cpu(), want), (targets.cpu() - want).abs().max()

    loss64, grad64, lab = _truth64(logits, want, labels, matched)
    assert abs(loss.item() - loss64) <= 1e-5 * abs(loss64)

    xr = logits.clone().requires_grad_(True)
    roi_heads.maskrcnn_loss(xr, proposals, masks, labels, matched).backward()
    ours, ref = x.grad.cpu(), xr.grad.cpu()
    err, ref_err = (ours.double() - grad64).abs().max().item(), (ref.double() - grad64).abs().max().item()
    assert err <= 2 * ref_err, (err, ref_err)
    off = torch.ones(ours.shape[:2], dtype=torch.bool)
    off[torch.arange(lab.shape[0]), lab] = False
    assert (ours[off] == 0).all() and (ref[off] == 0).all()
    assert not torch.signbit(ours[off]).any()


def test_bit_reproducible():
    logits, proposals, masks, labels, matched = _case("sizes")
    runs = []
    for _ in range(2):
        x = logits.clone().requires_grad_(True)
        loss, targets = det.maskrcnn_loss_op(x, proposals, masks, labels, matched)
        loss.backward()
        runs.append((loss.detach(), targets, x.grad))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("bad", ["match_past_gt", "negative_match", "label_past_classes"])
def test_bad_indices_give_nan(bad):
    logits, proposals, masks, labels, matched = _case("plain", C=7)
    matched = [m.clone() for m in matched]
    labels = [l.clone() for l in labels]
    if bad == "match_past_gt":
        matched[1][2] = masks[1].shape[0]
    elif bad == "negative_match":
        matched[1][2] = -1
    else:
        labels[1][:] = 7
    row = matched[0].shape[0] + 2
    bad_rows = torch.zeros(logits.shape[0], dtype=torch.bool)
    if bad == "label_past_classes":
        bad_rows[matched[0].shape[0]:] = True
    else:
        bad_rows[row] = True
    x = logits.clone().requires_grad_(True)
    loss, targets = det.maskrcnn_loss_op(x, proposals, masks, labels, matched)
    loss.backward()
    g, t = x.grad.cpu(), targets.cpu()
    assert torch.isnan(loss).item()
    assert torch.isnan(g[bad_rows]).all() and torch.isnan(t[bad_rows]).all()
    assert torch.isfinite(g[~bad_rows]).all() and torch.isfinite(t[~bad_rows]).all()


@pytest.mark.parametrize("name,forward,backward", [("plain", 2, 1), ("many", 3, 2)])
def test_no_host_sync_and_launch_counts(name, forward, backward):
    logits, proposals, masks, labels, matched = _case(name)

    def step():
        x = logits.clone().requires_grad_(True)
        loss, _ = det.maskrcnn_loss_op(x, proposals, masks, labels, matched)
        loss.backward()
        return x.grad

    step()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    n0 = _launches()
    loss, targets = torch.ops.vision_b200.maskrcnn_loss(logits, proposals, masks, labels, matched)
    n1 = _launches()
    torch.ops.vision_b200.maskrcnn_loss_backward(torch.ones((), device=DEV), logits, targets, labels, matched)
    n2 = _launches()
    assert (n1 - n0, n2 - n1) == (forward, backward)


def test_training_step_matches_the_reference_loss():
    """One training step of maskrcnn_resnet50_fpn with install() against install() without the maskrcnn_loss rebind; cuDNN
    is made deterministic so that each arm is bit-reproducible.  Only the mask loss differs: its value agrees to 1e-5
    relative, d loss / d mask_logits to 1e-6 of its largest entry, and every other loss is bit-identical.  As in the
    RetinaNet head-loss test, the untrained backbone's BatchNorm layers amplify those last-bit differences many-fold, so the
    parameter gradients are held to 2e-2 of each one's largest entry: far below what a wrong scale, a dropped image or a
    misplaced plane gives."""
    from torchvision.models.detection import maskrcnn_resnet50_fpn

    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    torch.manual_seed(0)
    model = maskrcnn_resnet50_fpn(weights=None, weights_backbone=None, min_size=480, max_size=640).to(DEV).train()
    gen = torch.Generator(device=DEV).manual_seed(1)
    images = [torch.rand(3, 480, 640, generator=gen, device=DEV) for _ in range(2)]
    targets = []
    for m in (5, 3):
        xy = torch.rand(m, 2, generator=gen, device=DEV) * 400
        boxes = torch.cat([xy, xy + 40 + torch.rand(m, 2, generator=gen, device=DEV) * 150], 1)
        masks = torch.zeros(m, 480, 640, dtype=torch.uint8, device=DEV)
        for j, b in enumerate(boxes.round().int().tolist()):
            masks[j, b[1] + 5:b[3] - 5, b[0] + 5:b[2] - 5] = 1
        targets.append({"boxes": boxes, "labels": torch.randint(1, 91, (m,), generator=gen, device=DEV), "masks": masks})
    state = copy.deepcopy(model.state_dict())
    seen = {}

    def keep_logits(module, inputs, output):
        output.retain_grad()
        seen["mask_logits"] = output

    model.roi_heads.mask_predictor.register_forward_hook(keep_logits)

    def step(rebind):
        model.load_state_dict(state)
        model.zero_grad(set_to_none=True)
        torch.manual_seed(2)                # the same proposal sampling (randperm) in both arms
        vision_b200.install()
        try:
            if not rebind:
                from vision_b200 import _install

                roi_heads.maskrcnn_loss = _install._state["orig_mask_loss"]
            losses = model(images, targets)
            sum(losses.values()).backward()
        finally:
            vision_b200.uninstall()
        return ({k: v.detach() for k, v in losses.items()}, seen["mask_logits"].grad.clone(),
                {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None})

    try:
        fused_losses, fused_g, fused_grads = step(True)
        ref_losses, ref_g, ref_grads = step(False)
    finally:
        torch.backends.cudnn.deterministic = False
    assert fused_losses.keys() == ref_losses.keys() and "loss_mask" in ref_losses
    for k in ref_losses:
        if k == "loss_mask":
            assert abs(fused_losses[k].item() - ref_losses[k].item()) <= 1e-5 * abs(ref_losses[k].item())
        else:
            assert torch.equal(fused_losses[k], ref_losses[k]), k
    assert (fused_g - ref_g).abs().max().item() <= 1e-6 * ref_g.abs().max().item()
    assert fused_grads.keys() == ref_grads.keys()
    for n, g in ref_grads.items():
        assert (fused_grads[n] - g).abs().max().item() <= 2e-2 * g.abs().max().item(), n
