"""deform_conv2d backward across the geometries and dtypes the forward accepts, against a float64 restatement of it.

The backward (torch_shim.cpp, deform_conv2d_backward) is two cuBLAS GEMMs around kernels of ours: dcol = W^T grad_out per
weight group, dcn_backward_inputs_kernel (grad_offset, grad_mask and, by default, grad_input scattered with atomics),
dcn_sample_columns_kernel (the sampled columns) and grad_weight = grad_out columns^T.  The batch runs in chunks of images
whose columns (plus, under torch.use_deterministic_algorithms, the per-image workspace of the gather) fit 2^30 bytes.  In
deterministic mode grad_input comes from bin, sort, cell records and dcn_grad_input_gather_kernel instead of the atomics.

Truth: `dcn_bwd_ref64`, all five gradients in float64 on the same rounded inputs, pinned on the CPU against the reference's
own CPU backward in float64.  Error scale: `dcn_bwd_mag64`, the same sums with every term replaced by its absolute value
(M, per element).  Every output element must satisfy |got - ref| <= c * M + tiny, tiny the dtype's smallest subnormal:

    fp64 1e-12, fp32 2^-16, fp16 8 * 2^-11, bf16 8 * 2^-8

except default-mode (atomic) grad_input at 16 bits, where every add rounds to 16 bits: (n_adds + 2) * u * M per element,
u = 2^-11 (fp16) or 2^-8 (bf16), n_adds the atomic adds into the element; the 2 are the rounding of dcol and of each term.
For fp16 the RoI tests' rule (max error at most 1.5x that of the reference's own fp16 CUDA backward) was tried and does not
hold with any headroom: both sides are a few random-order half roundings, and on the small border geometry oracle7 ours came
out 2.6x the reference's max error, while no fp16 case came above 0.53 of the analytic bound.

Worst ratio |got - ref| / bound over the matrix and the image chunks, all cases and both mask settings,
measured on an H100 80GB HBM3 (700 W power limit):
    dtype     mode       input  weight  offset    mask    bias
    float64   default  0.00039 0.00041 0.00028 0.00026       0
    float64   det      0.00038 0.00041 0.00028 0.00026       0
    float32   default    0.019   0.019   0.011  0.0087  0.0027
    float32   det        0.021   0.019   0.011  0.0092  0.0027
    float16   default     0.53    0.49    0.21    0.26   0.079
    float16   det         0.21    0.49    0.21    0.26   0.079
    bfloat16  default     0.61    0.29    0.22    0.21   0.086
    bfloat16  det         0.19    0.29    0.22    0.21   0.086
The analytic bounds of atomic 16-bit grad_input leave 1.9x (fp16) and 1.6x (bf16) headroom; they are not widened past
their analytic value.
"""
import zlib

import pytest
import torch

from test_dcn_backward_deterministic import deterministic
from test_dcn_geometry import CASES, CODE, ORACLE_GEOMETRIES, dcn_ref64, launched_kernel_names, make_inputs, out_size, worst_ratio

DEV = "cuda"
NAMES = ("input", "weight", "offset", "mask", "bias")
C_DTYPE = {torch.float64: 1e-12, torch.float32: 2.0 ** -16, torch.float16: 8 * 2.0 ** -11, torch.bfloat16: 8 * 2.0 ** -8}
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
CODE64 = {**CODE, torch.float64: 3}                                                 # VB200_F64


def tiny(dtype):
    f = torch.finfo(dtype)
    return f.smallest_normal * f.eps


# =============================== float64 restatement of the backward ===============================
def _sample_geometry(off_b, H, W, kh, kw, stride, padding, dilation, Ho, Wo):
    """One image's samples, each [OG, KK, P]: bilinear_interpolate's outer test, the fractions (lh, lw) and the four
    corners (flat index clamped into the image, inside-the-image flag, bilinear weight) in the order (hl, wl), (hl, wl + 1),
    (hl + 1, wl), (hl + 1, wl + 1).  The position is formed in fp64 for fp64 offsets and in fp32 otherwise, as the op does."""
    dev = off_b.device
    KK, P = kh * kw, Ho * Wo
    OG = off_b.shape[0] // (2 * KK)
    (sh, sw), (ph, pw), (dh, dw) = stride, padding, dilation
    pix = torch.arange(P, device=dev)
    oy, ox = pix // Wo, pix % Wo
    ti = torch.arange(kh, device=dev).repeat_interleave(kw)
    tj = torch.arange(kw, device=dev).repeat(kh)
    pos = torch.float64 if off_b.dtype == torch.float64 else torch.float32
    offv = off_b.reshape(OG, KK, 2, P).to(pos)
    y = ((oy[None, :] * sh - ph + ti[:, None] * dh).to(pos) + offv[:, :, 0]).double()
    x = ((ox[None, :] * sw - pw + tj[:, None] * dw).to(pos) + offv[:, :, 1]).double()
    inside = ~((y <= -1) | (y >= H) | (x <= -1) | (x >= W))
    hl, wl = torch.floor(y), torch.floor(x)
    lh, lw = y - hl, x - wl
    hh, hw = 1 - lh, 1 - lw
    hl, wl = hl.clamp(-2, H + 1).long(), wl.clamp(-2, W + 1).long()
    corners = []
    for cy, cx, wt in ((hl, wl, hh * hw), (hl, wl + 1, hh * lw), (hl + 1, wl, lh * hw), (hl + 1, wl + 1, lh * lw)):
        ok = (cy >= 0) & (cy <= H - 1) & (cx >= 0) & (cx <= W - 1)
        corners.append((cy.clamp(0, H - 1) * W + cx.clamp(0, W - 1), ok, wt))
    return inside, lh, lw, corners


def _dcn_bwd64(grad, x, off, w, mask=None, stride=(1, 1), padding=(0, 0), dilation=(1, 1)):
    """(gradients, magnitudes, n_adds) of deform_conv2d in float64 on x's device, one image at a time.

    gradients: grad_input, grad_weight, grad_offset, grad_mask (None without a mask), grad_bias.  magnitudes: the same five
    with every term of every sum replaced by its absolute value.  n_adds [B, C, H, W]: the number of nonzero terms
    scattered into each grad_input element (the default mode's atomic adds)."""
    f64 = torch.float64
    dev = x.device
    B, C, H, W = x.shape
    Co, Cg, kh, kw = w.shape
    G, KK = C // Cg, kh * kw
    OG = off.shape[1] // (2 * KK)
    cpo, cog = C // OG, Co // G
    Ho, Wo = grad.shape[2], grad.shape[3]
    P = Ho * Wo
    w2 = w.to(f64).reshape(G, cog, Cg * KK)
    z = lambda *s: torch.zeros(*s, dtype=f64, device=dev)
    gi, gim, adds = z(B, OG, cpo, H * W), z(B, OG, cpo, H * W), z(B, OG, H * W)
    go, gom = z(B, OG, KK, 2, P), z(B, OG, KK, 2, P)
    gm, gmm = z(B, OG, KK, P), z(B, OG, KK, P)
    gw, gwm = z(G, cog, Cg * KK), z(G, cog, Cg * KK)
    for b in range(B):
        inside, lh, lw, corners = _sample_geometry(off[b], H, W, kh, kw, stride, padding, dilation, Ho, Wo)
        g = grad[b].to(f64).reshape(G, cog, P)
        dcol = torch.einsum("gok,gop->gkp", w2, g).reshape(OG, cpo, KK, P)
        dcolm = torch.einsum("gok,gop->gkp", w2.abs(), g.abs()).reshape(OG, cpo, KK, P)
        m = mask[b].to(f64).reshape(OG, 1, KK, P) if mask is not None else torch.ones(OG, 1, KK, P, dtype=f64, device=dev)
        xs = x[b].to(f64).reshape(OG, cpo, H * W)
        v, wts = [], []
        for idx, ok, wt in corners:
            val = torch.gather(xs, 2, idx.reshape(OG, 1, KK * P).expand(OG, cpo, KK * P)).reshape(OG, cpo, KK, P)
            v.append(torch.where(ok[:, None], val, 0.0))
            wts.append(torch.where(ok & inside, wt, 0.0)[:, None])           # the blend and the scatter: inside samples only
        bil = sum(wk * vk for wk, vk in zip(wts, v))
        bilm = sum(wk.abs() * vk.abs() for wk, vk in zip(wts, v))
        gw += torch.einsum("gop,gkp->gok", g, (m * bil).reshape(G, Cg * KK, P))
        gwm += torch.einsum("gop,gkp->gok", g.abs(), (m.abs() * bilm).reshape(G, Cg * KK, P))
        gm[b], gmm[b] = (dcol * bil).sum(1), (dcolm * bilm).sum(1)
        # get_coordinate_weight, with no outer test: a sample on y = -1 has its row-0 corners
        hh, hw, lh, lw = (1 - lh)[:, None], (1 - lw)[:, None], lh[:, None], lw[:, None]
        md, mdm = m * dcol, m.abs() * dcolm
        go[b, :, :, 0] = (md * (hw * (v[2] - v[0]) + lw * (v[3] - v[1]))).sum(1)
        go[b, :, :, 1] = (md * (hh * (v[1] - v[0]) + lh * (v[3] - v[2]))).sum(1)
        a = [vk.abs() for vk in v]
        gom[b, :, :, 0] = (mdm * (hw.abs() * (a[2] + a[0]) + lw.abs() * (a[3] + a[1]))).sum(1)
        gom[b, :, :, 1] = (mdm * (hh.abs() * (a[1] + a[0]) + lh.abs() * (a[3] + a[2]))).sum(1)
        del v, a, bil, bilm
        for (idx, ok, wt), wk in zip(corners, wts):
            flat = idx.reshape(OG, 1, KK * P).expand(OG, cpo, KK * P)
            gi[b].scatter_add_(2, flat, (md * wk).reshape(OG, cpo, KK * P))
            gim[b].scatter_add_(2, flat, (mdm * wk.abs()).reshape(OG, cpo, KK * P))
            adds[b].scatter_add_(1, idx.reshape(OG, KK * P), (wk[:, 0] != 0).to(f64).reshape(OG, KK * P))
    g64 = grad.to(f64)
    shape_go, shape_gm = (B, OG * KK * 2, Ho, Wo), (B, OG * KK, Ho, Wo)
    grads = (gi.reshape(B, C, H, W), gw.reshape(Co, Cg, kh, kw), go.reshape(shape_go),
             gm.reshape(shape_gm) if mask is not None else None, g64.sum((0, 2, 3)))
    mags = (gim.reshape(B, C, H, W), gwm.reshape(Co, Cg, kh, kw), gom.reshape(shape_go),
            gmm.reshape(shape_gm) if mask is not None else None, g64.abs().sum((0, 2, 3)))
    n_adds = adds[:, :, None].expand(B, OG, cpo, H * W).reshape(B, C, H, W)
    return grads, mags, n_adds


def dcn_bwd_ref64(grad, x, off, w, mask=None, stride=(1, 1), padding=(0, 0), dilation=(1, 1)):
    """deform_conv2d's backward in float64 on x's device: (grad_input, grad_weight, grad_offset, grad_mask, grad_bias).

    dcol = W^T grad_out per weight group.  grad_input scatters mask * dcol * corner weight onto the live corners of every
    sample that passes bilinear_interpolate's outer test (-1 < y < H, -1 < x < W); grad_mask = sum over the offset group's
    channels of dcol * bilinear sample (inside samples only, None without a mask); grad_offset = sum of mask * dcol *
    get_coordinate_weight, with no outer test, as the reference's deformable_col2im_coord_kernel; grad_weight = grad_out
    columns^T; grad_bias = sum of grad_out.  The sample position is formed as dcn_ref64 forms it (fp32 for fp32 and 16-bit
    offsets), but in fp64 for fp64 offsets."""
    return _dcn_bwd64(grad, x, off, w, mask, stride, padding, dilation)[0]


def dcn_bwd_mag64(grad, x, off, w, mask=None, stride=(1, 1), padding=(0, 0), dilation=(1, 1)):
    """The sums of dcn_bwd_ref64 with every term replaced by its absolute value: the per-element error scale M."""
    return _dcn_bwd64(grad, x, off, w, mask, stride, padding, dilation)[1]


def bound_ratio(got, ref, mag, c, dtype):
    """max over elements of |got - ref| / (c * M + tiny): the check passes when this is at most 1."""
    return ((got.double() - ref).abs() / (c * mag + tiny(dtype))).max().item() if got.numel() else 0.0


def atomic16_ratio(got, ref, mag, n_adds, dtype):
    """bound_ratio of a grad_input scattered with 16-bit atomics: each of the n_adds adds into an element rounds the running
    sum (at most u M each), and dcol and every term round once more before they get there."""
    return ((got.double() - ref).abs() / ((n_adds + 2) * UNIT[dtype] * mag + tiny(dtype))).max().item() if got.numel() else 0.0


# =============================== CPU: pin the restatement ===============================
def _tv_backward(grad, x, off, w, m, b, s, p, d, use_mask):
    import torchvision  # noqa: F401  (registers torch.ops.torchvision)

    G, OG = x.shape[1] // w.shape[1], off.shape[1] // (2 * w.shape[2] * w.shape[3])
    mm = m if use_mask else torch.zeros(x.shape[0], 1, dtype=x.dtype, device=x.device)
    return torch.ops.torchvision._deform_conv2d_backward(grad, x, w, off, mm, b, *s, *p, *d, G, OG, use_mask)


def _grad_like(gen, B, Co, Ho, Wo, dtype=torch.float64, device="cpu"):
    return (torch.randn(B, Co, Ho, Wo, generator=gen) * 0.5).to(dtype).to(device)


@pytest.mark.parametrize("use_mask", [True, False], ids=["mask", "nomask"])
@pytest.mark.parametrize("geo", range(len(ORACLE_GEOMETRIES)))
def test_bwd_ref64_matches_reference_cpu(geo, use_mask):
    """Every gradient of the restatement against the reference's own CPU backward in float64, to 1e-12 of M."""
    B, C, H, W, Co, k, s, p, d, G, OG, _, bias, offs = ORACLE_GEOMETRIES[geo]
    gen = torch.Generator().manual_seed(200 + geo)
    x, off, w, b, m = make_inputs(gen, B, C, H, W, Co, k, s, p, d, G, OG, "randn", True, offs, dtype=torch.float64)
    Ho, Wo = out_size(H, k[0], s[0], p[0], d[0]), out_size(W, k[1], s[1], p[1], d[1])
    grad = _grad_like(gen, B, Co, Ho, Wo)
    mk = m if use_mask else None
    grads, mags, _ = _dcn_bwd64(grad, x, off, w, mk, s, p, d)
    want = _tv_backward(grad, x, off, w, m, b, s, p, d, use_mask)
    for name, got_, ref, mag in zip(NAMES, want, grads, mags):
        if ref is None:
            assert torch.equal(got_, torch.zeros_like(got_)), name
            continue
        assert got_.shape == ref.shape, name
        r = bound_ratio(got_, ref, mag, 1e-12, torch.float64)
        assert r <= 1, f"geometry {geo} grad_{name}: ratio {r:.3g}"
    assert (grads[0] != 0).any() and (grads[2] != 0).any()


def test_bwd_ref64_offset_gradient_on_the_border():
    """A tap exactly on y = -1 (zero offsets, padding 1) samples 0, yet its row-0 corners give it an offset gradient: the
    reference's grad_offset, unlike autograd through the forward's zero, is nonzero there."""
    gen = torch.Generator().manual_seed(3)
    x, off, w, b, m = make_inputs(gen, 1, 2, 5, 5, 2, (3, 3), (1, 1), (1, 1), (1, 1), 1, 1, "randn", True, "zero",
                                  dtype=torch.float64)
    grad = _grad_like(gen, 1, 2, 5, 5)
    go = dcn_bwd_ref64(grad, x, off, w, m, (1, 1), (1, 1), (1, 1))[2].reshape(9, 2, 5, 5)
    assert (go[0:3, 0, 0, 1:4].abs() > 0).all()                                    # taps of row i = 0 at output row 0: y = -1
    torch.testing.assert_close(go, _tv_backward(grad, x, off, w, m, b, (1, 1), (1, 1), (1, 1), True)[2].reshape(9, 2, 5, 5),
                               rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("geo", range(len(ORACLE_GEOMETRIES)))
def test_bwd_ref64_is_the_adjoint_of_dcn_ref64(geo):
    """The forward is linear in the input, the mask and the weights (offsets fixed), so <grad, out - bias> equals
    <grad_input, x>, <grad_mask, mask> and <grad_weight, w>, and <grad, bias> equals <grad_bias, bias>: ties the backward
    restatement to the forward one it must differentiate."""
    B, C, H, W, Co, k, s, p, d, G, OG, _, _, offs = ORACLE_GEOMETRIES[geo]
    gen = torch.Generator().manual_seed(300 + geo)
    x, off, w, b, m = make_inputs(gen, B, C, H, W, Co, k, s, p, d, G, OG, "randn", True, offs, dtype=torch.float64)
    out = dcn_ref64(x, off, w, None, s, p, d, m)
    grad = _grad_like(gen, *out.shape)
    gi, gw, _, gm, gb = dcn_bwd_ref64(grad, x, off.float(), w, m, s, p, d)          # fp32 positions, as dcn_ref64's
    lhs = (grad * out).sum().reshape(1)
    for rhs in ((gi * x).sum(), (gm * m).sum(), (gw * w).sum()):
        assert worst_ratio(rhs.reshape(1), lhs, 1e-12) <= 1, (lhs.item(), rhs.item())
    assert worst_ratio((gb * b).sum().reshape(1), (grad.sum((0, 2, 3)) * b).sum().reshape(1), 1e-12) <= 1


# =============================== GPU helpers ===============================
def _special_offsets(kind, gen, off, spec):
    """"huge": about a third of the offset coordinates set to +-2^31, +-3e9 or +-1e12, so (int)floor(y) overflows;
    "cell": every sample of every image at a random point inside the cell (7, 9) (fractions 0.2 ... 0.8)."""
    B, C, H, W, Co, (kh, kw), (sh, sw), (ph, pw), (dh, dw), G, OG = spec[:11]
    if kind == "huge":
        vals = torch.tensor([2.0 ** 31, -2.0 ** 31, 3e9, -3e9, 1e12, -1e12])
        pick = torch.rand(off.shape, generator=gen) < 0.3
        return torch.where(pick, vals[torch.randint(0, len(vals), off.shape, generator=gen)], off)
    Ho, Wo = off.shape[2], off.shape[3]
    ti = torch.arange(kh).repeat_interleave(kw).view(1, -1, 1, 1).float()
    tj = torch.arange(kw).repeat(kh).view(1, -1, 1, 1).float()
    oy = torch.arange(Ho).view(1, 1, Ho, 1).float()
    ox = torch.arange(Wo).view(1, 1, 1, Wo).float()
    ty = 7 + 0.2 + 0.6 * torch.rand(B, OG, kh * kw, Ho, Wo, generator=gen)
    tx = 9 + 0.2 + 0.6 * torch.rand(B, OG, kh * kw, Ho, Wo, generator=gen)
    dy = ty - (oy * sh - ph + ti * dh)
    dx = tx - (ox * sw - pw + tj * dw)
    return torch.stack((dy, dx), 3).reshape(off.shape)


def matrix_inputs(spec, dtype, seed, device=DEV):
    """(grad, x, off, w, mask, bias) of a matrix case in `dtype`: always a mask (the call decides whether it is used), a zero
    bias where the case has none."""
    B, C, H, W, Co, k, s, p, d, G, OG, _, bias, offs = spec
    gen = torch.Generator().manual_seed(seed)
    base = offs if offs in ("rand", "zero", "border", "leave") else "rand"
    x, off, w, b, m = make_inputs(gen, B, C, H, W, Co, k, s, p, d, G, OG, "randn", bias, base)
    if base != offs:
        off = _special_offsets(offs, gen, off, spec)
    if b is None:
        b = torch.zeros(Co)
    grad = _grad_like(gen, B, Co, out_size(H, k[0], s[0], p[0], d[0]), out_size(W, k[1], s[1], p[1], d[1]), torch.float32)
    return tuple(t.to(dtype).to(device) for t in (grad, x, off, w, m, b))


def _op(grad, x, off, w, m, b, s, p, d, use_mask):
    G, OG = x.shape[1] // w.shape[1], off.shape[1] // (2 * w.shape[2] * w.shape[3])
    mm = m if use_mask else torch.zeros(x.shape[0], 1, dtype=x.dtype, device=x.device)
    return torch.ops.vision_b200._deform_conv2d_backward(grad, x, w, off, mm, b, *s, *p, *d, G, OG, use_mask)


def launched_backward_kernels(fn, det):
    """(fn(), the kernel names the profiler recorded, the number of calls of fn), in deterministic mode when det.  The
    session is repeated, up to three times, while its trace lacks either of the two kernels every call launches: a trace
    that lost events says nothing about the gather kernel."""
    calls = [0]

    def counted():
        calls[0] += 1
        return fn()

    for _ in range(3):
        if det:
            with deterministic():
                out, names = launched_kernel_names(counted)
        else:
            out, names = launched_kernel_names(counted)
        if all(any(k in n for n in names) for k in ("dcn_backward_inputs_kernel", "dcn_sample_columns_kernel")):
            return out, names, calls[0]
    raise AssertionError(f"no complete profiler trace in three sessions: {sorted(names)}")


def check_outputs(label, got, truth, dtype, det):
    """Asserts the bounds of the module docstring on the five outputs; returns {output name: worst ratio}.
    truth = (gradients, magnitudes, n_adds) of _dcn_bwd64."""
    grads, mags, n_adds = truth
    c = C_DTYPE[dtype]
    ratios = {}
    for name, a, ref, mag in zip(NAMES, got, grads, mags):
        assert a.dtype == dtype, f"{label} grad_{name}: dtype {a.dtype}"
        if ref is None:                                                           # grad_mask without a mask
            assert torch.equal(a, torch.zeros_like(a)), f"{label} grad_{name}"
            continue
        assert a.shape == ref.shape, f"{label} grad_{name}: shape {tuple(a.shape)} != {tuple(ref.shape)}"
        if det:
            assert torch.isfinite(a).all(), f"{label} grad_{name}: not written in full"
        if name == "input" and not det and dtype in UNIT:
            r = atomic16_ratio(a, ref, mag, n_adds, dtype)
        else:
            r = bound_ratio(a, ref, mag, c, dtype)
        ratios[name] = r
        print(f"RATIO {str(dtype)[6:]} {'det' if det else 'default'} {name} {label} {r:.3g}")
        assert r <= 1, f"{label} grad_{name}: worst ratio {r:.3g}"
    return ratios


# =============================== GPU: geometry x dtype x mode x mask ===============================
# B, C, H, W, Co, (kh, kw), stride, pad, dil, G, OG, mask (unused: both settings run), bias, offsets
MATRIX = {name: spec for name, (spec, _, _) in CASES.items()}
MATRIX.update({f"oracle{i}": spec for i, spec in enumerate(ORACLE_GEOMETRIES)})
MATRIX.update({
    "out1x1": (2, 8, 3, 4, 6, (3, 3), (1, 2), (0, 0), (1, 1), 2, 2, "randn", True, "rand"),           # a 1 x 1 output
    # offsets of +-2^31 and beyond, where (int)floor(y) saturates: the sample has no live corner at all
    "huge_off": (2, 16, 9, 11, 8, (3, 3), (1, 1), (1, 1), (1, 1), 2, 4, "randn", True, "huge"),
    # all 9 x 256 samples of an image in one cell: 2304 terms into each of its four pixels per channel
    "one_cell": (2, 64, 16, 16, 32, (3, 3), (1, 1), (1, 1), (1, 1), 1, 1, "randn", True, "cell"),
})
DTYPES = [torch.float64, torch.float32, torch.float16, torch.bfloat16]
# fp16 cannot hold an offset of 2^31
MATRIX_PARAMS = [(n, t) for n in MATRIX for t in DTYPES if not (n == "huge_off" and t == torch.float16)]


@pytest.mark.gpu
@pytest.mark.parametrize("use_mask", [True, False], ids=["mask", "nomask"])
@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
@pytest.mark.parametrize("name,dtype", MATRIX_PARAMS, ids=[f"{n}-{str(t)[6:]}" for n, t in MATRIX_PARAMS])
def test_backward_matrix(vb, name, dtype, det, use_mask):
    spec = MATRIX[name]
    s, p, d = spec[6], spec[7], spec[8]
    grad, x, off, w, m, b = matrix_inputs(spec, dtype, seed=zlib.crc32(name.encode()) % 10_000)
    label = f"{name}/{'mask' if use_mask else 'nomask'}"
    before = vb.launch_count()
    got, kernels, calls = launched_backward_kernels(lambda: _op(grad, x, off, w, m, b, s, p, d, use_mask), det)
    # per call (one chunk, one pass): the inputs kernel and the column sampler, plus bin, sort, cell start, records and gather
    assert vb.launch_count() - before == calls * (7 if det else 2), f"{label}: {vb.launch_count() - before} launches in {calls} calls"
    gathered = any("dcn_grad_input_gather_kernel" in k for k in kernels)
    assert gathered == det, f"{label}: dcn_grad_input_gather_kernel launched: {gathered}, deterministic: {det}"
    truth = _dcn_bwd64(grad, x, off, w, m if use_mask else None, s, p, d)
    check_outputs(label, got, truth, dtype, det)
    if name == "one_cell":
        assert ((got[0] != 0).sum(dim=(2, 3)) <= 4).all()
    assert truth[0][0].abs().max() > 0 or name == "huge_off"


# =============================== GPU: image chunks ===============================
def chunk_images(dtype, B, C, H, W, k, OG, det):
    """Images per chunk of the backward: the columns of one image (C * KK * HWo elements) plus, in deterministic mode, the
    gather's workspace for one image, within 2^30 bytes."""
    from vision_b200 import _lib

    KK, HWo = k * k, out_size(H, k, 1, 1, 1) * out_size(W, k, 1, 1, 1)
    ws =_lib.core().vb200_deform_conv2d_backward_inputs_workspace_bytes(CODE64[dtype], 1, C, H, W, k, k, 1, 1, 1, 1, 1, 1, OG) if det else 0
    assert not det or ws > 0
    per_img = C * KK * HWo * torch.empty(0, dtype=dtype).element_size() + ws
    return max(1, min(B, (1 << 30) // per_img))


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
@pytest.mark.parametrize("dtype,C", [(torch.float32, 256), (torch.bfloat16, 512)], ids=["float32", "bfloat16"])
def test_backward_image_chunks(vb, dtype, C, det):
    """3 x 3 over a 128 x 128 map (128 x 128 output): 151 MB of columns per image at C = 256 fp32 or C = 512 bf16, so nine
    images run as chunks of 7 and 2 (deterministic: 6 and 3, the workspace counts too).  grad_weight accumulates across
    the chunks; every output is checked against the fp64 truth, and in deterministic mode every image's grad_input,
    grad_offset and grad_mask against a call with that image alone, bit for bit."""
    B, H, W, Co, G, OG = 9, 128, 128, 16, 2, 2
    chunk = chunk_images(dtype, B, C, H, W, 3, OG, det)
    assert 1 < chunk < B and B % chunk, (chunk, B)
    spec = (B, C, H, W, Co, (3, 3), (1, 1), (1, 1), (1, 1), G, OG, "randn", True, "rand")
    grad, x, off, w, m, b = matrix_inputs(spec, dtype, seed=C + det)
    one = (1, 1)
    if det:
        with deterministic():
            got = _op(grad, x, off, w, m, b, one, one, one, True)
            singles = [_op(grad[i:i + 1], x[i:i + 1], off[i:i + 1], w, m[i:i + 1], b, one, one, one, True) for i in range(B)]
        for i, single in enumerate(singles):
            for k_ in (0, 2, 3):
                assert torch.equal(got[k_][i:i + 1], single[k_]), (i, NAMES[k_])
        del singles
    else:
        got = _op(grad, x, off, w, m, b, one, one, one, True)
    truth = _dcn_bwd64(grad, x, off, w, m, one, one, one)
    check_outputs(f"chunks{chunk}", got, truth, dtype, det)


# =============================== GPU: operand layouts ===============================
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_backward_layouts_bit_equal(vb, dtype):
    """A channels-last input, a non-contiguous grad (a transposed view) and an offset that is a channel slice of a larger
    tensor give the bits of their contiguous copies: all five outputs in deterministic mode; in the default mode all but
    the atomically scattered grad_input."""
    spec = (2, 64, 13, 15, 128, (3, 3), (1, 1), (1, 1), (1, 1), 1, 2, "randn", True, "rand")
    grad, x, off, w, m, b = matrix_inputs(spec, dtype, seed=17)
    xcl = x.contiguous(memory_format=torch.channels_last)
    gnc = grad.transpose(2, 3).contiguous().transpose(2, 3)
    big = torch.zeros(off.shape[0], 2 * off.shape[1], *off.shape[2:], dtype=dtype, device=DEV)
    osl = big[:, off.shape[1]:]
    osl.copy_(off)
    assert not (xcl.is_contiguous() or gnc.is_contiguous() or osl.is_contiguous())
    one = (1, 1)
    with deterministic():
        plain = _op(grad, x, off, w, m, b, one, one, one, True)
        strided = _op(gnc, xcl, osl, w, m, b, one, one, one, True)
    for name, a, c in zip(NAMES, plain, strided):
        assert torch.isfinite(a).all() and torch.equal(a, c), name
    plain = _op(grad, x, off, w, m, b, one, one, one, True)
    strided = _op(gnc, xcl, osl, w, m, b, one, one, one, True)
    for name, a, c in list(zip(NAMES, plain, strided))[1:]:
        assert torch.equal(a, c), name


# =============================== GPU: through torchvision's autograd ===============================
AUTOGRAD_SPECS = {
    "c64": (2, 64, 11, 13, 128, (3, 3), (1, 1), (1, 1), (1, 1), 1, 2, "randn", True, "border"),
    "out1x1": (3, 16, 4, 5, 8, (4, 5), (1, 1), (0, 0), (1, 1), 2, 4, "randn", True, "rand"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("use_mask", [True, False], ids=["mask", "nomask"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32], ids=lambda t: str(t)[6:])
@pytest.mark.parametrize("case", list(AUTOGRAD_SPECS))
def test_installed_torchvision_autograd(vb, case, dtype, use_mask):
    """After install(), torchvision.ops.deform_conv2d(...).backward() runs on these kernels and its five gradients meet
    the bounds of the matrix (16-bit grad_input: the analytic (n_adds + 2) u M, which holds for fp16 as for bf16)."""
    import torchvision

    spec = AUTOGRAD_SPECS[case]
    s, p, d = spec[6], spec[7], spec[8]
    grad, x, off, w, m, b = matrix_inputs(spec, dtype, seed=zlib.crc32(case.encode()) % 1000)
    ins = [t.clone().requires_grad_(True) for t in (x, off, w, b, m)]
    was = vb.installed()
    vb.install()
    try:
        before = vb.launch_count()
        out = torchvision.ops.deform_conv2d(ins[0], ins[1], ins[2], ins[3], s, p, d, ins[4] if use_mask else None)
        out.backward(grad)
        assert vb.launch_count() >= before + 3                    # forward, backward inputs, columns
    finally:
        if not was:
            vb.uninstall()
    got = (ins[0].grad, ins[2].grad, ins[1].grad, ins[4].grad if use_mask else torch.zeros_like(m), ins[3].grad)
    truth = _dcn_bwd64(grad, x, off, w, m if use_mask else None, s, p, d)
    grads, mags, n_adds = truth
    for name, a, ref, mag in zip(NAMES, got, grads, mags):
        if ref is None:
            assert torch.equal(a, torch.zeros_like(a)) or a is None, name
            continue
        assert a.shape == ref.shape and a.dtype == dtype, name
        if name == "input" and dtype in UNIT:
            r = atomic16_ratio(a, ref, mag, n_adds, dtype)
        else:
            r = bound_ratio(a, ref, mag, C_DTYPE[dtype], dtype)
        assert r <= 1, f"{case} {dtype} grad_{name}: worst ratio {r:.3g}"


@pytest.mark.gpu
def test_installed_torchvision_autograd_empty_batch(vb):
    """B = 0: the backward returns empty input / offset / mask gradients and zero weight / bias gradients."""
    import torchvision

    x = torch.zeros(0, 8, 6, 7, device=DEV, requires_grad=True)
    off = torch.zeros(0, 18, 6, 7, device=DEV, requires_grad=True)
    m = torch.zeros(0, 9, 6, 7, device=DEV, requires_grad=True)
    w = torch.randn(4, 8, 3, 3, device=DEV, requires_grad=True)
    b = torch.randn(4, device=DEV, requires_grad=True)
    was = vb.installed()
    vb.install()
    try:
        out = torchvision.ops.deform_conv2d(x, off, w, b, padding=1, mask=m)
        assert out.shape == (0, 4, 6, 7)
        out.sum().backward()
    finally:
        if not was:
            vb.uninstall()
    assert x.grad.shape == x.shape and off.grad.shape == off.shape and m.grad.shape == m.shape
    assert torch.equal(w.grad, torch.zeros_like(w)) and torch.equal(b.grad, torch.zeros_like(b))
