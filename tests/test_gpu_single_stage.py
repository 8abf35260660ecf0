"""GPU suite: RetinaNet / FCOS / SSD / SSDLite postprocess_detections through the fused select + decode + NMS pipeline
against the same method run with vision_b200 uninstalled (the installed wheel's kernels), bit for bit.

torch.topk does not order equal scores; our rule is (score desc, index asc).  Every bit-exact case therefore asserts, as a
precondition, that the top k + 1 passing scores of every segment are distinct; seeds are taken in a fixed order until one
satisfies it."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
tv = pytest.importorskip("torchvision")
if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from torchvision.models.detection import _utils as det_utils  # noqa: E402
from torchvision.models.detection.fcos import FCOS  # noqa: E402
from torchvision.models.detection.retinanet import RetinaNet  # noqa: E402
from torchvision.models.detection.ssd import SSD  # noqa: E402

import vision_b200  # noqa: E402

DEV = "cuda"
PRIOR = -math.log((1 - 0.01) / 0.01)          # -4.595: the classification head's bias


def _launches():
    vision_b200._lib.load_ops()
    return torch.ops.vision_b200._launch_count()


def _bare(cls, coder, **attrs):
    m = cls.__new__(cls)
    m.box_coder = coder
    for k, v in attrs.items():
        setattr(m, k, v)
    return m


def retinanet(**kw):
    a = dict(score_thresh=0.05, topk_candidates=1000, nms_thresh=0.5, detections_per_img=300)
    a.update(kw)
    return _bare(RetinaNet, det_utils.BoxCoder(weights=(1.0, 1.0, 1.0, 1.0)), **a)


def fcos(**kw):
    a = dict(score_thresh=0.2, topk_candidates=1000, nms_thresh=0.6, detections_per_img=100)
    a.update(kw)
    return _bare(FCOS, det_utils.BoxLinearCoder(normalize_by_size=True), **a)


def ssd(**kw):
    a = dict(score_thresh=0.01, topk_candidates=400, nms_thresh=0.45, detections_per_img=200)
    a.update(kw)
    return _bare(SSD, det_utils.BoxCoder(weights=(10.0, 10.0, 5.0, 5.0)), **a)


def _anchors(n, gen, h, w):
    xy = torch.rand(n, 2, generator=gen, device=DEV) * torch.tensor([w, h], device=DEV, dtype=torch.float32)
    wh = torch.exp(torch.rand(n, 2, generator=gen, device=DEV) * 3.5 + 2.5)
    return torch.cat([xy - wh / 2, xy + wh / 2], 1)


def fpn_inputs(shapes, C=91, A_loc=9, mu=PRIOR, sd=1.0, ctrness=False, seed=0, pad=(800, 1088)):
    """Head outputs as RetinaNet / FCOS hand them over: per-level views split from [N, sum A, *] (retinanet.py:640-655).
    Each (image, level) gets a stratified N(mu, sd) sample - the quantiles of n equal-probability strata, randomly placed -
    so the top scores of a level are distinct (independent draws put two equal scores into the top 1000 of an 11 M-element
    level about once per image).  FCOS ctrness is constant per level (sigmoid 1.0 or 0.5, exact factors) for the same reason;
    the end-to-end FCOS test covers per-anchor ctrness."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    levels = [math.ceil(pad[0] / s) * math.ceil(pad[1] / s) * A_loc for s in (8, 16, 32, 64, 128)]
    N, total = len(shapes), sum(levels)
    cls = torch.empty(N, total, C, device=DEV)
    for n in range(N):
        for lv, rows in zip(cls[n].split(levels), levels):
            m = rows * C
            q = (torch.randperm(m, generator=gen, device=DEV).double() + 0.5) / m
            lv.copy_((torch.special.ndtri(q) * sd + mu).float().view(rows, C))
    reg = torch.randn(N, total, 4, generator=gen, device=DEV) * 0.5
    head = {"cls_logits": list(cls.split(levels, 1)), "bbox_regression": list(reg.split(levels, 1))}
    if ctrness:
        head["bbox_ctrness"] = [torch.full((N, a, 1), 20.0 if l % 2 == 0 else 0.0, device=DEV) for l, a in enumerate(levels)]
    anchors = [list(_anchors(total, gen, *pad).split(levels)) for _ in shapes]
    return head, anchors, list(shapes)


def ssd_inputs(shapes, A=8732, C=91, sd=2.0, seed=0, size=300):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    N = len(shapes)
    head = {"cls_logits": torch.randn(N, A, C, generator=gen, device=DEV) * sd,
            "bbox_regression": torch.randn(N, A, 4, generator=gen, device=DEV) * 0.5}
    return head, [_anchors(A, gen, size, size) for _ in shapes], list(shapes)


def _segment_scores(model, head):
    """Passing scores of every segment, restated with the reference's tensor ops."""
    if isinstance(model, SSD):
        p = torch.softmax(head["cls_logits"], -1)
        for n in range(p.shape[0]):
            for c in range(1, p.shape[2]):
                s = p[n, :, c]
                yield s[s > model.score_thresh]
        return
    for l, lg in enumerate(head["cls_logits"]):
        for n in range(lg.shape[0]):
            s = torch.sigmoid(lg[n])
            if isinstance(model, FCOS):
                s = torch.sqrt(s * torch.sigmoid(head["bbox_ctrness"][l][n]))
            s = s.flatten()
            yield s[s > model.score_thresh]


def _distinct_top(model, head):
    for s in _segment_scores(model, head):
        v = s.topk(min(model.topk_candidates + 1, s.numel())).values
        if v.numel() > 1 and bool((v[1:] == v[:-1]).any()):
            return False
    return True


def _with_distinct_top(model, make, seeds=range(16)):
    for seed in seeds:
        inputs = make(seed)
        if _distinct_top(model, inputs[0]):
            return inputs
    pytest.fail("precondition: no seed gives distinct top-(k+1) scores in every segment")


def _run_both(model, inputs):
    head, anchors, shapes = inputs
    vision_b200.uninstall()
    ref = type(model).postprocess_detections(model, head, anchors, shapes)
    vision_b200.install()
    try:
        before = _launches()
        got = type(model).postprocess_detections(model, head, anchors, shapes)
        after = _launches()
    finally:
        vision_b200.uninstall()
    assert after > before, "the fused kernels did not run"
    return ref, got


def _assert_equal(ref, got):
    assert len(ref) == len(got)
    for r, g in zip(ref, got):
        assert g["boxes"].shape == r["boxes"].shape and g["boxes"].dtype == r["boxes"].dtype
        assert g["labels"].dtype == torch.int64 and g["scores"].dtype == r["scores"].dtype
        for k in ("boxes", "scores", "labels"):
            assert torch.equal(g[k], r[k]), k


SHAPES = {1: [(800, 1088)], 2: [(800, 1066), (704, 1088)], 8: [(800, 1088), (800, 1066), (750, 1088), (800, 960),
                                                               (640, 1088), (800, 1024), (720, 1000), (800, 800)]}
SSD_SHAPES = {1: [(300, 300)], 2: [(300, 300), (280, 300)], 8: [(300, 300)] * 4 + [(300, 290), (260, 300), (300, 300), (240, 300)]}


@pytest.mark.parametrize("batch", [1, 2, 8])
def test_retinanet_parity(batch):
    m = retinanet()
    ref, got = _run_both(m, _with_distinct_top(m, lambda s: fpn_inputs(SHAPES[batch], seed=s)))
    _assert_equal(ref, got)
    assert sum(r["boxes"].shape[0] for r in ref) > 0


@pytest.mark.parametrize("batch", [1, 2, 8])
def test_fcos_parity(batch):
    m = fcos()
    ref, got = _run_both(m, _with_distinct_top(m, lambda s: fpn_inputs(SHAPES[batch], A_loc=1, ctrness=True, seed=s)))
    _assert_equal(ref, got)
    assert sum(r["boxes"].shape[0] for r in ref) > 0


@pytest.mark.parametrize("batch", [1, 2, 8])
def test_ssd300_parity(batch):
    m = ssd()
    ref, got = _run_both(m, _with_distinct_top(m, lambda s: ssd_inputs(SSD_SHAPES[batch], seed=s)))
    _assert_equal(ref, got)
    assert sum(r["boxes"].shape[0] for r in ref) > 0


@pytest.mark.parametrize("batch", [1, 2, 8])
def test_ssdlite320_parity(batch):
    m = ssd(score_thresh=0.001, topk_candidates=300, nms_thresh=0.55, detections_per_img=300)
    shapes = ([(320, 320), (300, 320)] * 4)[:batch]
    ref, got = _run_both(m, _with_distinct_top(m, lambda s: ssd_inputs(shapes, A=3234, seed=s, size=320)))
    _assert_equal(ref, got)


def test_low_threshold_many_outputs_bit_exact():
    """Thousands of sigmoid / sqrt / decode results reach the output."""
    shapes = [(800, 1088), (704, 1088)]
    for m, kw in ((retinanet(score_thresh=0.0, topk_candidates=1000, nms_thresh=0.7, detections_per_img=6000), {}),
                  (fcos(score_thresh=0.0, topk_candidates=1000, nms_thresh=0.7, detections_per_img=5000), dict(A_loc=1, ctrness=True))):
        ref, got = _run_both(m, _with_distinct_top(m, lambda s: fpn_inputs(shapes, C=20, mu=-8.0, sd=2.0, seed=100 + s, **kw)))
        _assert_equal(ref, got)
        assert min(r["boxes"].shape[0] for r in ref) > 2000


def test_nothing_passes():
    m = retinanet(score_thresh=0.999)
    ref, got = _run_both(m, fpn_inputs(SHAPES[2], mu=-12.0, sd=0.5))
    for g in got:
        assert g["boxes"].shape == (0, 4) and g["scores"].shape == (0,) and g["labels"].shape == (0,)
        assert g["labels"].dtype == torch.int64 and g["boxes"].dtype == torch.float32
    _assert_equal(ref, got)


def test_fewer_pass_than_topk():
    m = retinanet()
    inputs = _with_distinct_top(m, lambda s: fpn_inputs(SHAPES[2], mu=-7.0, sd=1.0, seed=s))
    assert all(s.numel() < m.topk_candidates for s in _segment_scores(m, inputs[0]))
    ref, got = _run_both(m, inputs)
    _assert_equal(ref, got)
    assert 0 < sum(r["boxes"].shape[0] for r in ref)


def test_scores_exactly_at_threshold_are_dropped():
    """1500 (anchor, class) probabilities of exactly 0.25.  top-k and detections_per_img exceed every candidate count and
    NMS hardly suppresses, so under `>=` they would reach the output; `>` must drop them."""
    m = ssd(score_thresh=0.25, topk_candidates=2000, nms_thresh=0.99, detections_per_img=8000)

    def make(seed):
        head, anchors, shapes = ssd_inputs(SSD_SHAPES[1], C=4, A=2000, seed=seed)
        head["cls_logits"][0, :500] = 0.0          # four equal logits: softmax gives exactly 0.25 (a power of two)
        return head, anchors, shapes

    inputs = _with_distinct_top(m, make)
    p = torch.softmax(inputs[0]["cls_logits"], -1)
    assert bool((p[0, :500] == 0.25).all())
    assert all(s.numel() + 500 <= m.topk_candidates for s in _segment_scores(m, inputs[0]))
    ref, got = _run_both(m, inputs)
    _assert_equal(ref, got)
    assert got[0]["scores"].numel() > 0 and not bool((got[0]["scores"] <= 0.25).any())


@pytest.mark.parametrize("thresh", [-0.0, -1e-60, 0.0])
def test_zero_thresholds(thresh):
    """-0.0 (and a negative double that rounds to -0.0f) passes every positive score, as +0.0 does."""
    m = retinanet(score_thresh=thresh)
    ref, got = _run_both(m, _with_distinct_top(m, lambda s: fpn_inputs(SHAPES[2], seed=s)))
    _assert_equal(ref, got)
    m = ssd(score_thresh=thresh)
    ref, got = _run_both(m, _with_distinct_top(m, lambda s: ssd_inputs(SSD_SHAPES[1], seed=s)))
    _assert_equal(ref, got)


class _MyCoder(det_utils.BoxCoder):
    pass


def _fallback_cases():
    small = dict(pad=(128, 160), C=5)
    yield "retinanet_fp16", retinanet(), fpn_inputs([(128, 160)], **small), torch.float16
    yield "ssd_fp16", ssd(), ssd_inputs([(300, 300)], A=500, C=6), torch.float16
    yield "retinanet_subclassed_coder", _bare(RetinaNet, _MyCoder(weights=(1.0, 1.0, 1.0, 1.0)), score_thresh=0.05, topk_candidates=1000,
                                              nms_thresh=0.5, detections_per_img=300), fpn_inputs([(128, 160)], **small), None
    yield "ssd_subclassed_coder", _bare(SSD, _MyCoder(weights=(10.0, 10.0, 5.0, 5.0)), score_thresh=0.01, topk_candidates=400, nms_thresh=0.45,
                                        detections_per_img=200), ssd_inputs([(300, 300)], A=500, C=6), None
    yield "fcos_unnormalized", _bare(FCOS, det_utils.BoxLinearCoder(normalize_by_size=False), score_thresh=0.2, topk_candidates=1000,
                                     nms_thresh=0.6, detections_per_img=100), fpn_inputs([(128, 160)], A_loc=1, ctrness=True, **small), None
    yield "retinanet_topk_above_capacity", retinanet(topk_candidates=vision_b200.detection.SINGLE_STAGE_MAX_TOPK + 1), \
        fpn_inputs([(128, 160)], **small), None
    yield "retinanet_strided_logits", retinanet(), fpn_inputs([(128, 160)], **small), "strided"


@pytest.mark.parametrize("label", [c[0] for c in _fallback_cases()])
def test_uncovered_cuda_inputs_take_the_reference_body(label, monkeypatch):
    """CUDA inputs the fused kernel does not cover go to the original method (the fused op is never called)."""
    from vision_b200 import detection as det

    _, model, (head, anchors, shapes), how = next(c for c in _fallback_cases() if c[0] == label)
    if how == torch.float16:
        head = {k: [t.half() for t in v] if isinstance(v, list) else v.half() for k, v in head.items()}
        anchors = [[a.half() for a in x] if isinstance(x, list) else x.half() for x in anchors]
    elif how == "strided":       # last dimension not dense
        head["cls_logits"] = [t.transpose(1, 2).contiguous().transpose(1, 2) for t in head["cls_logits"]]
    vision_b200.uninstall()
    expected = type(model).postprocess_detections(model, head, anchors, shapes)

    def refuse(*a, **k):
        raise AssertionError("the fused path must not be taken for these inputs")

    monkeypatch.setattr(det, "single_stage_postprocess", refuse)
    vision_b200.install()
    try:
        got = type(model).postprocess_detections(model, head, anchors, shapes)
    finally:
        vision_b200.uninstall()
    _assert_equal(expected, got)


@pytest.mark.parametrize("many", [True, False])
def test_ssd_vanilla_and_trick_paths(many):
    """More than 25 000 candidates take the reference's per-class (vanilla) batched_nms, fewer the coordinate trick."""
    m = ssd(score_thresh=0.005 if many else 0.1, topk_candidates=400)
    inputs = _with_distinct_top(m, lambda s: ssd_inputs(SSD_SHAPES[1], sd=1.0 if many else 2.0, seed=20 + s))
    n_cand = sum(min(m.topk_candidates, s.numel()) for s in _segment_scores(m, inputs[0]))
    assert (n_cand > 25000) == many
    ref, got = _run_both(m, inputs)
    _assert_equal(ref, got)


def _restated_candidates(model, head, anchors, shapes):
    """The reference's selection with ties broken by index (torch.sort(stable=True)), then decode and clip."""
    out = []
    for n, hw in enumerate(shapes):
        boxes, scores, labels = [], [], []
        for l, lg in enumerate(head["cls_logits"]):
            C = lg.shape[-1]
            s = torch.sigmoid(lg[n]).flatten()
            idx = torch.where(s > model.score_thresh)[0]
            order = torch.sort(s[idx], stable=True, descending=True)[1][: model.topk_candidates]
            idx = idx[order]
            a = idx // C
            b = model.box_coder.decode_single(head["bbox_regression"][l][n][a], anchors[n][l][a])
            boxes.append(tv.ops.clip_boxes_to_image(b, hw))
            scores.append(s[idx])
            labels.append(idx % C)
        out.append((torch.cat(boxes), torch.cat(scores), torch.cat(labels)))
    return out


def _rows(b, s, l):
    t = torch.cat([b.double(), s.double()[:, None], l.double()[:, None]], 1)
    for col in reversed(range(t.shape[1])):
        t = t[torch.sort(t[:, col], stable=True)[1]]
    return t


def test_ties_follow_score_then_index():
    """Quantised logits: most scores tie.  NMS is switched off (IoU > 1 never holds) so the output is the candidate set."""
    m = retinanet(score_thresh=0.05, topk_candidates=300, nms_thresh=1.0, detections_per_img=100000)
    head, anchors, shapes = fpn_inputs(SHAPES[2], C=8, seed=7)
    head["cls_logits"] = [torch.round(t * 2) / 2 for t in head["cls_logits"]]
    ref, got = _run_both(m, (head, anchors, shapes))
    for r, g, (cb, cs, cl) in zip(ref, got, _restated_candidates(m, head, anchors, shapes)):
        assert torch.equal(torch.sort(g["scores"])[0], torch.sort(r["scores"])[0])
        assert torch.equal(_rows(g["boxes"], g["scores"], g["labels"]), _rows(cb, cs, cl))


def _head_outputs(model, imgs):
    """The head outputs the model hands to postprocess_detections."""
    seen = {}

    def capture(head_outputs, anchors, image_shapes):
        seen["head"] = head_outputs
        return type(model).postprocess_detections(model, head_outputs, anchors, image_shapes)

    model.postprocess_detections = capture
    try:
        model(imgs)
    finally:
        del model.postprocess_detections
    return seen["head"]


def _e2e(model, sizes):
    """Images are drawn seed by seed until the head's top k + 1 scores of every segment are distinct (the precondition of a
    bit-exact comparison), then the model runs with and without install()."""
    model = model.eval().to(DEV)
    with torch.no_grad():
        vision_b200.uninstall()
        for seed in range(8):
            torch.manual_seed(seed)
            imgs = [torch.rand(3, h, w, device=DEV) for h, w in sizes]
            if _distinct_top(model, _head_outputs(model, imgs)):
                break
        else:
            pytest.fail("precondition: no seed gives distinct top-(k+1) scores in every segment")
        ref = model(imgs)
        vision_b200.install()
        try:
            before = _launches()
            got = model(imgs)
            assert _launches() > before
        finally:
            vision_b200.uninstall()
    _assert_equal(ref, got)
    return ref


def test_retinanet_resnet50_fpn_end_to_end():
    from torchvision.models.detection import retinanet_resnet50_fpn

    torch.manual_seed(0)
    # topk_candidates 100: equal scores in the top k + 1 become ~k^2 times rarer (the parity tests cover k = 1000)
    m = retinanet_resnet50_fpn(weights=None, weights_backbone=None, score_thresh=0.011, topk_candidates=100)
    torch.nn.init.normal_(m.head.classification_head.cls_logits.weight, std=0.05)    # spread the fresh head's scores
    ref = _e2e(m, [(480, 640), (512, 384)])
    assert sum(r["boxes"].shape[0] for r in ref) > 0


def test_fcos_resnet50_fpn_end_to_end():
    from torchvision.models.detection import fcos_resnet50_fpn

    torch.manual_seed(0)
    m = fcos_resnet50_fpn(weights=None, weights_backbone=None, score_thresh=0.011)
    torch.nn.init.normal_(m.head.classification_head.cls_logits.weight, std=0.05)
    ref = _e2e(m, [(480, 640), (512, 384)])
    assert sum(r["boxes"].shape[0] for r in ref) > 0


def test_ssdlite320_mobilenet_v3_large_end_to_end():
    from torchvision.models.detection import ssdlite320_mobilenet_v3_large

    torch.manual_seed(0)
    m = ssdlite320_mobilenet_v3_large(weights=None, weights_backbone=None, score_thresh=0.005).to(DEV)
    # With default BatchNorm statistics a fresh backbone gives the same features for every input and location, so every
    # class scores exactly 1/91.  One train-mode pass over random images sets the statistics, and the scores vary.
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.reset_running_stats()
                mod.momentum = None
        m.train()
        m.head(list(m.backbone(torch.rand(4, 3, 320, 320, device=DEV)).values()))
        m.eval()
    ref = _e2e(m, [(320, 320), (300, 400)])
    assert sum(r["boxes"].shape[0] for r in ref) > 0
