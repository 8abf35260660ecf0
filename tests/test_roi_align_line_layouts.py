"""roi_align's line kernel (7x7 bins, sampling_ratio 2) on RoI sets that drive each of its lane arrangements - lanes along x or
along y, picked per RoI by the geometry kernel - and its edge cases: tiny, wide and short, tall and narrow, large square RoIs,
RoIs hanging outside the map, bad batch indices, two images, odd widths.  Each set is checked against the oracle on the line
path, and the fused MultiScaleRoIAlign and peer-destination instantiations of the same kernel against the line path's output."""
import importlib.util
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32_TOL = dict(rtol=1e-5, atol=1e-5)
SCALE = 0.25


def _model():
    spec = importlib.util.spec_from_file_location("roi_line_model", os.path.join(ROOT, "tools", "roi_line_model.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _boxes(g, k, wmin, wmax, hmin, hmax, img_w, img_h, lo=0.0, hi=1.0):
    w = g.uniform(wmin, wmax, k)
    h = g.uniform(hmin, hmax, k)
    x1 = g.uniform(lo, hi, k) * img_w - w * lo
    y1 = g.uniform(lo, hi, k) * img_h - h * lo
    return np.stack([x1, y1, x1 + w, y1 + h], 1)


def roi_sets():
    """name -> (B, H, W, rois [K, 5] in image coordinates at SCALE)"""
    g = np.random.default_rng(7)
    out = {}

    def add(name, B, H, W, boxes, batch=None):
        k = boxes.shape[0]
        b = g.integers(0, B, k) if batch is None else batch
        out[name] = (B, H, W, np.concatenate([b[:, None].astype(np.float32), boxes.astype(np.float32)], 1))

    H, W = 60, 88
    iw, ih = W / SCALE, H / SCALE
    add("small", 1, H, W, _boxes(g, 160, 2, 24, 2, 24, iw, ih))
    add("wide_short", 1, H, W, _boxes(g, 160, 200, 340, 4, 16, iw, ih))
    add("tall_narrow", 1, H, W, _boxes(g, 160, 4, 16, 140, 230, iw, ih))
    add("large_square", 1, H, W, _boxes(g, 160, 130, 240, 130, 240, iw, ih))
    add("outside", 1, H, W, _boxes(g, 160, 20, 300, 20, 300, iw, ih, lo=-0.4, hi=1.3))
    bad = g.integers(0, 2, 160)
    bad[::5] = -1
    bad[1::5] = 2
    add("bad_batch", 2, H, W, _boxes(g, 160, 10, 200, 10, 200, iw, ih), batch=bad)
    add("two_images", 2, H, W, _boxes(g, 160, 10, 300, 10, 300, iw, ih))
    add("odd_width_53", 1, 41, 53, _boxes(g, 160, 4, 200, 4, 160, 53 / SCALE, 41 / SCALE))
    add("odd_width_97", 2, 35, 97, _boxes(g, 160, 8, 380, 4, 140, 97 / SCALE, 35 / SCALE))
    return out


SETS = roi_sets()


def test_every_lane_arrangement_is_exercised():
    """the model's restatement of the geometry kernel's choice picks both lane axes across the sets (and both within the
    sets meant to force them), so the GPU tests below run every arrangement"""
    m = _model()
    picks = {name: m.lane_axis_is_y(r, SCALE, H, W) for name, (B, H, W, r) in SETS.items()}
    assert picks["wide_short"].mean() > 0.5            # lanes along y: a line across a wide RoI spans more than 32 banks
    assert picks["tall_narrow"].mean() < 0.1           # lanes along x, for the same reason
    assert not picks["small"].any()                    # both are conflict-free: ties go to x
    for name in ("large_square", "outside", "two_images", "odd_width_97"):
        assert 0 < picks[name].mean() < 1, name


class _force_line:
    def __enter__(self):
        from vision_b200 import _lib

        self.old = os.environ.get("VB200_ROI_ALIGN_PATH")
        os.environ["VB200_ROI_ALIGN_PATH"] = "line"
        _lib.core().vb200_reload_env()

    def __exit__(self, *a):
        from vision_b200 import _lib

        if self.old is None:
            os.environ.pop("VB200_ROI_ALIGN_PATH", None)
        else:
            os.environ["VB200_ROI_ALIGN_PATH"] = self.old
        _lib.core().vb200_reload_env()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SETS))
def test_line_kernel_instantiations_on_roi_set(vb, oracle, name):
    B, H, W, rois = SETS[name]
    C = 12
    x = np.random.default_rng(len(name)).standard_normal((B, C, H, W)).astype(np.float32)
    xd, rd = torch.from_numpy(x).cuda(), torch.from_numpy(rois).cuda()
    with _force_line():
        got = torch.ops.vision_b200.roi_align(xd, rd, SCALE, 7, 7, 2, False)
        ok = (rois[:, 0] >= 0) & (rois[:, 0] < B)
        safe = rois.copy()
        safe[~ok, 0] = 0
        want = oracle.roi_align(x, safe, 7, SCALE, 2, False)
        np.testing.assert_allclose(got.cpu().numpy()[ok], want[ok], **F32_TOL)
        assert not got[torch.from_numpy(~ok).cuda()].any(), "RoIs with a batch index outside [0, B) produce zeros"

        # the peer-destination instantiation: three local buffers stand in for the peers' slots
        n = got.numel()
        bufs = [torch.full((n + 32,), -3.0, device="cuda") for _ in range(3)]
        torch.ops.vision_b200.roi_align_gather(xd, rd, [b.data_ptr() + 64 for b in bufs], 0, SCALE, 7, 7, 2, False)
        for b in bufs:
            assert torch.equal(b[16:16 + n].view(got.shape), got)
            assert bool((b[:16] == -3).all()) and bool((b[16 + n:] == -3).all())

    # the fused MultiScaleRoIAlign instantiation with one level: every RoI maps to it (k_min == k_max)
    out, levels = torch.ops.vision_b200.multiscale_roi_align([xd], rd, [SCALE], 7, 7, 2, 2, 2, 224.0, 4.0, 1e-6)
    assert bool((levels == 0).all())
    assert torch.equal(out, got)
