"""deform_conv2d forward across the geometries its three kernels accept, against a float64 restatement of the op.

The forward has three kernels: deform_conv2d_tc_kernel (bf16 / fp16 on wgmma, BN = 256 or 128 output channels per CTA),
deform_conv2d_tc3_kernel (fp32 as a bf16x3 split on wgmma) and deform_conv2d_simt_kernel (everything else).  Every case
here names the path it was written for and asserts it through the packed-weight query of the C ABI, so a change of the
eligibility rules cannot silently turn the matrix into SIMT-only coverage.

Bounds (BASELINE.json north_star): |got - ref| <= 1e-5 (1 + |ref|) for fp32, 1e-2 (1 + |ref|) for bf16 / fp16, where ref is
`dcn_ref64` evaluated on the same rounded inputs.  Weights are scaled by 1 / sqrt(c_in_g * KK), so the output is O(1) and
the bound means the same thing at every depth.

`dcn_ref64` is pinned on the CPU (no GPU needed) against the reference's golden vectors and the CPU oracle."""
import math
import os
import re
import zlib

import numpy as np
import pytest
import torch

DEV = "cuda"
F32_BOUND, F16_BOUND = 1e-5, 1e-2
CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}     # VB200_F32 / VB200_F16 / VB200_BF16


class force_env:
    """Sets a VB200_* override for the duration of a block (the library reads its overrides once, not per call)."""

    def __init__(self, key, val):
        self.key, self.val = key, val

    def __enter__(self):
        from vision_b200 import _lib

        self.old = os.environ.get(self.key)
        os.environ[self.key] = self.val
        _lib.core().vb200_reload_env()

    def __exit__(self, *a):
        from vision_b200 import _lib

        if self.old is None:
            os.environ.pop(self.key, None)
        else:
            os.environ[self.key] = self.old
        _lib.core().vb200_reload_env()


# =============================== float64 restatement ===============================
def out_size(n, k, s, p, d):
    return (n + 2 * p - (d * (k - 1) + 1)) // s + 1


def dcn_ref64(x, off, w, bias=None, stride=(1, 1), padding=(0, 0), dilation=(1, 1), mask=None, pixels=None):
    """deform_conv2d forward in float64 on x's device.

    The sample position of tap (i, j) at output pixel (oy, ox) is oy * stride_h - pad_h + i * dil_h + offset_h (and the
    same along w).  It is formed in fp32, as the op forms it for fp32 and 16-bit inputs alike; everything after it is
    fp64.  Bilinear sampling follows the reference's bilinear_interpolate: zero when h <= -1 or H <= h (or the same for
    w); otherwise the corners floor(h), floor(h) + 1 (and along w), each counted only when inside the image, with weights
    hh * hw, hh * lw, lh * hw, lh * lw.  The sample is multiplied by the mask, then contracted with each weight group.

    `pixels` (1-D int64 of flat output indices oy * out_w + ox) restricts the evaluation to those pixels of every image;
    the result is then [B, c_out, len(pixels)], otherwise [B, c_out, out_h, out_w]."""
    dev = x.device
    B, C, H, W = x.shape
    Co, Cg, kh, kw = w.shape
    G, KK = C // Cg, kh * kw
    OG = off.shape[1] // (2 * KK)
    cpo = C // OG
    (sh, sw), (ph, pw), (dh, dw) = stride, padding, dilation
    Ho, Wo = out_size(H, kh, sh, ph, dh), out_size(W, kw, sw, pw, dw)
    pix = torch.arange(Ho * Wo, device=dev) if pixels is None else pixels.to(dev)
    P = pix.numel()
    oy, ox = pix // Wo, pix % Wo
    ti = torch.arange(kh, device=dev).repeat_interleave(kw)       # tap = i * kw + j
    tj = torch.arange(kw, device=dev).repeat(kh)
    offv = off.reshape(B, OG, KK, 2, Ho * Wo)[..., pix].float()     # [B, OG, KK, 2, P]
    base_y = (oy[None, :] * sh - ph + ti[:, None] * dh).float()     # [KK, P], exact integers
    base_x = (ox[None, :] * sw - pw + tj[:, None] * dw).float()
    y = (base_y + offv[:, :, :, 0]).double()                        # fp32 add, then fp64
    xx = (base_x + offv[:, :, :, 1]).double()
    inside = ~((y <= -1) | (y >= H) | (xx <= -1) | (xx >= W))
    hl, wl = torch.floor(y), torch.floor(xx)
    lh, lw = y - hl, xx - wl
    hh, hw = 1 - lh, 1 - lw
    hl, wl = hl.clamp(-2, H + 1).long(), wl.clamp(-2, W + 1).long()
    xs = x.reshape(B, OG, cpo, H * W)
    val = torch.zeros(B, OG, cpo, KK, P, dtype=torch.float64, device=dev)
    for cy, cx, wt in ((hl, wl, hh * hw), (hl, wl + 1, hh * lw), (hl + 1, wl, lh * hw), (hl + 1, wl + 1, lh * lw)):
        ok = inside & (cy >= 0) & (cy <= H - 1) & (cx >= 0) & (cx <= W - 1)
        idx = (cy.clamp(0, H - 1) * W + cx.clamp(0, W - 1)).reshape(B, OG, 1, KK * P).expand(B, OG, cpo, KK * P)
        v = torch.gather(xs, 3, idx).double().reshape(B, OG, cpo, KK, P)
        val += v * torch.where(ok, wt, torch.zeros_like(wt))[:, :, None]
    if mask is not None:
        val = val * mask.reshape(B, OG, KK, Ho * Wo)[..., pix].double()[:, :, None]
    cols = val.reshape(B, G, Cg * KK, P)
    out = torch.einsum("gok,bgkp->bgop", w.double().reshape(G, Co // G, Cg * KK), cols).reshape(B, Co, P)
    if bias is not None:
        out = out + bias.double()[None, :, None]
    return out if pixels is not None else out.reshape(B, Co, Ho, Wo)


def worst_ratio(got, ref, bound):
    """max over elements of |got - ref| / (bound * (1 + |ref|)): the check passes when this is at most 1."""
    g, r = got.double(), ref.double()
    return ((g - r).abs() / (bound * (1 + r.abs()))).max().item()


def make_inputs(gen, B, C, H, W, Co, k, stride, pad, dil, G, OG, mask="randn", bias=True, offsets="rand", dtype=torch.float32,
                device="cpu", act=None):
    """Seeded fp32 inputs rounded to `dtype`.  offsets: "rand" (N(0, 2), crosses every border of small maps), "zero",
    "border" (integer offsets onto -1, 0, H - 1, H and the same along w, plus half-pixel ones next to them) or "leave"
    (offsets of +-H / +-W, mostly outside the image).  Weights ~ N(0, 1 / (c_in_g * KK))."""
    kh, kw = k
    Ho, Wo = out_size(H, kh, stride[0], pad[0], dil[0]), out_size(W, kw, stride[1], pad[1], dil[1])
    KK = kh * kw
    x = torch.randn(B, C, H, W, generator=gen) if act is None else act(torch.randn(B, C, H, W, generator=gen))
    wt = torch.randn(Co, C // G, kh, kw, generator=gen) / math.sqrt(C // G * KK)
    if offsets == "zero":
        off = torch.zeros(B, OG * 2 * KK, Ho, Wo)
    elif offsets == "rand":
        off = torch.randn(B, OG * 2 * KK, Ho, Wo, generator=gen) * 2
    elif offsets == "leave":
        sgn = torch.randint(0, 2, (B, OG * KK, 2, Ho, Wo), generator=gen) * 2 - 1
        frac = torch.rand(B, OG * KK, 2, Ho, Wo, generator=gen)
        off = (sgn * (torch.tensor([H, W]).view(1, 1, 2, 1, 1) + frac - 0.5)).reshape(B, OG * 2 * KK, Ho, Wo)
    elif offsets == "border":
        ti = torch.arange(kh).repeat_interleave(kw)
        tj = torch.arange(kw).repeat(kh)
        base_y = torch.arange(Ho)[None, :] * stride[0] - pad[0] + ti[:, None] * dil[0]          # [KK, Ho]
        base_x = torch.arange(Wo)[None, :] * stride[1] - pad[1] + tj[:, None] * dil[1]          # [KK, Wo]
        ty_choices = torch.tensor([-1.0, 0.0, H - 1.0, float(H), -0.5, H - 0.5, -2.0, H + 1.0])
        tx_choices = torch.tensor([-1.0, 0.0, W - 1.0, float(W), -0.5, W - 0.5, -2.0, W + 1.0])
        ty = ty_choices[torch.randint(0, 8, (B, OG, KK, Ho, Wo), generator=gen)]
        tx = tx_choices[torch.randint(0, 8, (B, OG, KK, Ho, Wo), generator=gen)]
        oy_ = ty - base_y[None, None, :, :, None]
        ox_ = tx - base_x[None, None, :, None, :]
        off = torch.stack((oy_, ox_), dim=3).reshape(B, OG * 2 * KK, Ho, Wo)
    else:
        raise ValueError(offsets)
    m = torch.randn(B, OG * KK, Ho, Wo, generator=gen) if mask == "randn" else None
    b = torch.randn(Co, generator=gen) if bias else None
    cast = lambda t: None if t is None else t.to(dtype).to(device)
    return cast(x), cast(off), cast(wt), cast(b), cast(m)


# =============================== CPU: pin the restatement ===============================
def test_ref64_matches_reference_golden(golden):
    sh, sw, ph, pw, dh, dw = [int(v) for v in golden["dcn_args"]]
    t = lambda k: torch.from_numpy(golden[k])
    for key, mask in (("dcn_out_mask", t("dcn_mask")), ("dcn_out_nomask", None)):
        ref = dcn_ref64(t("dcn_x"), t("dcn_off"), t("dcn_w"), t("dcn_b"), (sh, sw), (ph, pw), (dh, dw), mask)
        want = torch.from_numpy(golden[key])
        assert ref.shape == want.shape
        assert worst_ratio(want, ref, 2e-6) <= 1, f"worst ratio {worst_ratio(want, ref, 2e-6):.3g}"


# B, C, H, W, Co, (kh, kw), stride, pad, dil, G, OG, mask, bias, offsets
ORACLE_GEOMETRIES = [
    (2, 6, 5, 4, 4, (3, 2), (2, 1), (1, 0), (2, 1), 2, 3, "randn", True, "rand"),      # the reference's test geometry
    (1, 8, 9, 11, 4, (2, 5), (1, 2), (0, 2), (3, 1), 4, 2, "randn", True, "rand"),     # kh != kw, mixed stride / dilation
    (2, 4, 12, 7, 6, (5, 2), (2, 2), (2, 0), (2, 2), 1, 1, None, True, "rand"),
    (1, 6, 6, 8, 6, (3, 3), (1, 1), (1, 1), (1, 1), 3, 2, "randn", False, "border"),   # exact -1, H - 1, H landings
    (2, 4, 7, 5, 4, (2, 3), (1, 1), (2, 1), (1, 2), 2, 4, "randn", True, "leave"),     # offsets leave the image
    (1, 4, 5, 9, 2, (1, 1), (3, 2), (0, 0), (1, 1), 2, 4, None, False, "rand"),
    (1, 6, 7, 7, 6, (3, 3), (1, 1), (2, 2), (1, 1), 3, 6, None, True, "zero"),          # zero offsets onto -1 / -2
    (2, 6, 8, 6, 3, (4, 3), (1, 2), (2, 1), (1, 1), 3, 2, "randn", True, "border"),    # 2 offset groups over 3 groups
]


@pytest.mark.parametrize("geo", range(len(ORACLE_GEOMETRIES)))
def test_ref64_matches_oracle(oracle, geo):
    B, C, H, W, Co, k, s, p, d, G, OG, mask, bias, offs = ORACLE_GEOMETRIES[geo]
    gen = torch.Generator().manual_seed(100 + geo)
    x, off, w, b, m = make_inputs(gen, B, C, H, W, Co, k, s, p, d, G, OG, mask, bias, offs)
    ref = dcn_ref64(x, off, w, b, s, p, d, m)
    n = lambda t: None if t is None else t.numpy()
    want = torch.from_numpy(oracle.deform_conv2d(n(x), n(off), n(w), n(b), s, p, d, n(m)))
    r = worst_ratio(want, ref, 2e-6)
    assert r <= 1, f"geometry {geo}: worst ratio {r:.3g}"
    assert ref.abs().max() > 0.1


def test_ref64_pixel_subset_matches_full():
    gen = torch.Generator().manual_seed(7)
    x, off, w, b, m = make_inputs(gen, 2, 6, 9, 7, 4, (3, 2), (1, 2), (1, 1), (2, 1), 2, 3)
    full = dcn_ref64(x, off, w, b, (1, 2), (1, 1), (2, 1), m)
    pix = torch.tensor([0, 5, 17, full.shape[2] * full.shape[3] - 1])
    sub = dcn_ref64(x, off, w, b, (1, 2), (1, 1), (2, 1), m, pixels=pix)
    torch.testing.assert_close(sub, full.flatten(2)[:, :, pix], rtol=1e-12, atol=1e-12)   # contraction order may differ


# =============================== GPU helpers ===============================
def align256(n):
    return (n + 255) // 256 * 256


def dcn_path(dtype, c_in, c_out, kh, kw, groups, offset_groups):
    """The forward kernel this shape takes, read from the packed-weight size the C ABI reports for it: 0 bytes for SIMT,
    2 bytes per weight for the 16-bit tensor-core kernel, 6 (three bf16 splits) for the fp32 one."""
    from vision_b200 import _lib

    n = _lib.core().vb200_deform_conv2d_packed_weight_bytes(CODE[dtype], c_in, c_out, kh, kw, groups, offset_groups)
    K = c_out * c_in * kh * kw
    if n == 0:
        return "simt"
    if n == align256(K * 2):
        return "tc"
    if n == align256(K * 6):
        return "tc3"
    raise AssertionError(f"unexpected packed-weight size {n}")


def launched_kernel_names(fn):
    """Runs fn under torch.profiler: (its result, the names of the events it recorded, device kernels among them).

    The profiler now and then delivers no device activity at all for a short session; fn (deterministic) then runs
    again, up to three times.  A session that recorded device kernels is never retried, whatever it found."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    for _ in range(3):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        events = prof.events()
        if any(e.device_type == DeviceType.CUDA for e in events):
            break
    return out, {e.name for e in events}


def launched_forward_kernels(fn):
    """Runs fn under torch.profiler and names the deform_conv2d forward kernels it launched: "tc256" / "tc128" for
    deform_conv2d_tc_kernel with BN = 256 / 128 output channels per CTA (its second template argument), "tc3" for
    deform_conv2d_tc3_kernel, "simt" for deform_conv2d_simt_kernel.  The packed-weight query tells the path class only;
    BN shows in the kernel's name alone."""
    out, names = launched_kernel_names(fn)
    labels = set()
    for name in names:
        bn = re.search(r"deform_conv2d_tc_kernel<[^,]*,[^0-9]*(\d+)", name) or re.search(r"deform_conv2d_tc_kernelI\w+?Li(\d+)E", name)
        if bn:
            labels.add("tc" + bn.group(1))
        elif "deform_conv2d_tc3_kernel" in name:
            labels.add("tc3")
        elif "deform_conv2d_simt_kernel" in name:
            labels.add("simt")
    return out, labels


def bound_of(dtype):
    return F32_BOUND if dtype == torch.float32 else F16_BOUND


def path_class(kernel):
    return "tc" if kernel in ("tc256", "tc128") else kernel


def run_case(vb, dtype, spec, expect, label, seed):
    """expect: the forward kernel the shape is written for (tc256 / tc128 / tc3 / simt)."""
    B, C, H, W, Co, k, s, p, d, G, OG, mask, bias, offs = spec
    path = dcn_path(dtype, C, Co, k[0], k[1], G, OG)
    assert path == path_class(expect), f"{label}: expected the {expect} path, the shape takes {path}"
    gen = torch.Generator().manual_seed(seed)
    x, off, w, b, m = make_inputs(gen, B, C, H, W, Co, k, s, p, d, G, OG, mask, bias, offs, dtype=dtype, device=DEV)
    before = vb.launch_count()
    got, kernels = launched_forward_kernels(lambda: vb.ops.deform_conv2d(x, off, w, b, s, p, d, m))
    assert vb.launch_count() > before
    assert kernels == {expect}, f"{label}: expected {expect}, launched {kernels}"
    ref = dcn_ref64(x, off, w, b, s, p, d, m)
    assert got.shape == ref.shape and got.dtype == dtype
    r = worst_ratio(got, ref, bound_of(dtype))
    print(f"{label} {str(dtype)[6:]} [{expect}] worst ratio {r:.3g}")
    assert r <= 1, f"{label} {dtype} [{expect}]: worst |got - ref| / (bound (1 + |ref|)) = {r:.3g}"
    return got


# =============================== GPU: geometry matrix ===============================
# name: (B, C, H, W, Co, (kh, kw), stride, pad, dil, G, OG, mask, bias, offsets), kernel for 16-bit, kernel for fp32
CASES = {
    # 1x1: KK = 1, n_q (1 per 64 channels) below the stage count; 7 x 9 = 63 pixels (< 128, odd: scalar epilogue)
    "k1x1_b3_63px": ((3, 64, 7, 9, 128, (1, 1), (1, 1), (0, 0), (1, 1), 1, 1, "randn", True, "rand"), "tc128", "tc3"),
    # 2x5 / 5x2, stride (2, 1) and 2, dilation (1, 3) and 2, padding (0, 2) / (2, 0); partial last tile
    "k2x5_s21_d13": ((1, 128, 27, 29, 256, (2, 5), (2, 1), (0, 2), (1, 3), 1, 1, "randn", True, "rand"), "tc256", "tc3"),
    "k5x2_s2_d2_p20": ((3, 64, 31, 17, 128, (5, 2), (2, 2), (2, 0), (2, 2), 1, 1, None, True, "rand"), "tc128", "tc3"),
    # 3x3 on non-square maps: 851 pixels (not a multiple of 8) and 960 (a multiple of 8, partial last tile)
    "k3x3_37x23": ((3, 64, 37, 23, 256, (3, 3), (1, 1), (1, 1), (1, 1), 1, 1, "randn", False, "rand"), "tc256", "tc3"),
    "k3x3_24x40_p2": ((1, 64, 22, 38, 128, (3, 3), (1, 1), (2, 2), (1, 1), 1, 1, "randn", True, "rand"), "tc128", "tc3"),
    # offset groups on the tensor cores: 64 channels each (16-bit and fp32), c_out 384 = three BN = 128 tiles, 512 = two BN = 256
    "og2_c128_co384": ((3, 128, 19, 13, 384, (3, 3), (1, 1), (1, 1), (1, 1), 1, 2, "randn", True, "rand"), "tc128", "tc3"),
    "og4_c256_co512": ((2, 256, 13, 21, 512, (3, 3), (2, 1), (1, 1), (1, 2), 1, 4, "randn", True, "rand"), "tc256", "tc3"),
    # 32 channels per offset group and c_in 32 / 96: tc3 only (the 16-bit kernel needs 64 per group)
    "og2_c64_cpo32": ((2, 64, 15, 11, 128, (3, 3), (1, 1), (1, 1), (1, 1), 1, 2, "randn", True, "rand"), "simt", "tc3"),
    "og4_c128_cpo32": ((1, 128, 12, 17, 256, (3, 3), (1, 1), (1, 1), (1, 1), 1, 4, "randn", True, "rand"), "simt", "tc3"),
    "c32": ((2, 32, 14, 10, 128, (3, 3), (1, 1), (1, 1), (1, 1), 1, 1, "randn", True, "rand"), "simt", "tc3"),
    "c96": ((1, 96, 10, 19, 256, (3, 3), (1, 1), (1, 1), (1, 1), 1, 1, "randn", True, "rand"), "simt", "tc3"),
    # kernel-size boundaries: KK 20 (last BN = 256, last tc3), 21 (BN = 128; fp32 SIMT), 24 (last tc), 25 (SIMT)
    "k4x5_kk20": ((1, 64, 19, 23, 256, (4, 5), (1, 1), (2, 2), (1, 1), 1, 1, "randn", True, "rand"), "tc256", "tc3"),
    "k3x7_kk21": ((1, 64, 17, 25, 256, (3, 7), (1, 1), (1, 3), (1, 1), 1, 1, "randn", True, "rand"), "tc128", "simt"),
    "k4x6_kk24": ((2, 64, 13, 15, 128, (4, 6), (1, 1), (2, 2), (1, 1), 1, 1, "randn", True, "rand"), "tc128", "simt"),
    "k5x5_kk25": ((1, 64, 16, 12, 128, (5, 5), (1, 1), (2, 2), (1, 1), 1, 1, "randn", True, "rand"), "simt", "simt"),
    # 11x11: KK = 121 is past the single-table limit of the SIMT kernel (106 taps)
    "k11x11_kk121": ((1, 32, 23, 20, 128, (11, 11), (1, 1), (5, 5), (1, 1), 1, 1, "randn", True, "rand"), "simt", "simt"),
    # offsets: zero with padding (taps exactly on -1 and -2), integer ones onto the borders, +-H out of the image
    "zero_off_p2": ((2, 64, 12, 14, 128, (3, 3), (1, 1), (2, 2), (1, 1), 1, 1, None, False, "zero"), "tc128", "tc3"),
    "border_off": ((2, 64, 11, 13, 256, (3, 3), (1, 1), (1, 1), (1, 1), 1, 1, "randn", True, "border"), "tc256", "tc3"),
    "border_off_og2": ((1, 128, 9, 14, 128, (2, 3), (1, 2), (1, 0), (2, 1), 1, 2, "randn", False, "border"), "tc128", "tc3"),
    "leave_off": ((2, 64, 10, 15, 128, (3, 3), (1, 1), (1, 1), (1, 1), 1, 1, "randn", True, "leave"), "tc128", "tc3"),
    # SIMT at real sizes: groups 2 / 4 with offset groups straddling them, cout_g 160 / 136, per-group K 675 (not % 16)
    "g2_og3_coutg160": ((2, 150, 13, 17, 320, (3, 3), (1, 1), (1, 1), (1, 1), 2, 3, "randn", True, "rand"), "simt", "simt"),
    "g4_og3_coutg136": ((1, 96, 16, 11, 544, (3, 2), (2, 1), (1, 0), (1, 2), 4, 3, "randn", True, "rand"), "simt", "simt"),
    "g1_coutg200": ((2, 40, 14, 9, 200, (3, 3), (1, 1), (1, 1), (1, 1), 1, 1, "randn", True, "border"), "simt", "simt"),
}
DTYPES = [torch.bfloat16, torch.float16, torch.float32]


def _expected(name, dtype):
    return CASES[name][2] if dtype == torch.float32 else CASES[name][1]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda t: str(t)[6:])
@pytest.mark.parametrize("name", list(CASES))
def test_forward_matrix_default_path(vb, name, dtype):
    run_case(vb, dtype, CASES[name][0], _expected(name, dtype), name, seed=zlib.crc32(name.encode()) % 10_000)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda t: str(t)[6:])
@pytest.mark.parametrize("name", list(CASES))
def test_forward_matrix_forced_simt(vb, name, dtype):
    with force_env("VB200_DCN_PATH", "simt"):
        run_case(vb, dtype, CASES[name][0], "simt", name + "/forced", seed=zlib.crc32(name.encode()) % 10_000)


# =============================== GPU: staging variants ===============================
@pytest.mark.gpu
@pytest.mark.parametrize("dtype,H,W", [(torch.bfloat16, 14, 12), (torch.bfloat16, 9, 11), (torch.float16, 13, 15),
                                       (torch.float32, 14, 12), (torch.float32, 9, 11)])
def test_staging_variants_bit_identical(vb, dtype, H, W):
    """A channels-last input (no staging copy) and an input whose storage starts one element past an aligned address
    (for 16-bit types a 2-byte offset: the scalar NCHW -> NHWC kernel) give the plain call's output bit for bit, at an
    even H * W (16-bit: the vectorised staging kernel) and an odd one (the scalar kernel)."""
    C, Co = 128, 256
    want_path = "tc3" if dtype == torch.float32 else "tc"
    assert dcn_path(dtype, C, Co, 3, 3, 1, 2) == want_path
    gen = torch.Generator().manual_seed(H * W)
    x, off, w, b, m = make_inputs(gen, 2, C, H, W, Co, (3, 3), (1, 1), (1, 1), (1, 1), 1, 2, dtype=dtype, device=DEV)
    plain = vb.ops.deform_conv2d(x, off, w, b, 1, 1, 1, m)
    r = worst_ratio(plain, dcn_ref64(x, off, w, b, (1, 1), (1, 1), (1, 1), m), bound_of(dtype))
    assert r <= 1, f"worst ratio {r:.3g}"
    xcl = x.contiguous(memory_format=torch.channels_last)
    assert not xcl.is_contiguous()
    assert torch.equal(vb.ops.deform_conv2d(xcl, off, w, b, 1, 1, 1, m), plain)
    buf = torch.empty(x.numel() + 1, dtype=dtype, device=DEV)
    xo = buf[1:].view(x.shape)
    xo.copy_(x)
    assert xo.is_contiguous() and xo.data_ptr() % 16 != 0
    assert dtype == torch.float32 or xo.data_ptr() % 4 == 2      # 16-bit: not 4-byte aligned, the scalar staging kernel
    assert torch.equal(vb.ops.deform_conv2d(xo, off, w, b, 1, 1, 1, m), plain)


# =============================== GPU: fp32 depth sweep (tc3) ===============================
DEPTHS = [(64, (3, 3)), (256, (3, 3)), (512, (3, 3)), (1024, (3, 3)), (1024, (2, 5))]     # K = 576 ... 10240


@pytest.mark.gpu
@pytest.mark.parametrize("act", ["normal", "relu4"])
def test_fp32_depth_sweep(vb, act):
    """fp32 on the bf16x3 tensor-core kernel at K = c_in * KK up to 10240: activations N(0, 1), or |N(0, 4)| like a
    post-ReLU feature map, weights N(0, 1 / K)."""
    fn = None if act == "normal" else (lambda t: (t * 4).abs())
    worst = {}
    for C, k in DEPTHS:
        K = C * k[0] * k[1]
        assert dcn_path(torch.float32, C, 128, k[0], k[1], 1, 1) == "tc3"
        gen = torch.Generator().manual_seed(K)
        x, off, w, b, _ = make_inputs(gen, 1, C, 16, 16, 128, k, (1, 1), (1, 1), (1, 1), 1, 1, None, True, "rand",
                                      dtype=torch.float32, device=DEV, act=fn)
        got = vb.ops.deform_conv2d(x, off, w, b, 1, 1, 1, None)
        ref = dcn_ref64(x, off, w, b, (1, 1), (1, 1), (1, 1), None)
        worst[K] = (worst_ratio(got, ref, F32_BOUND) * F32_BOUND, (got.double() - ref).abs().max().item())
        print(f"fp32 depth {act} K={K}: max |err| / (1 + |ref|) = {worst[K][0]:.3g}, max |err| = {worst[K][1]:.3g}")
    bad = {K: v for K, v in worst.items() if v[0] > F32_BOUND}
    assert not bad, f"over 1e-5 (1 + |ref|): {bad}"


# =============================== GPU: 32-bit corner offsets of the tensor-core gather ===============================
@pytest.mark.gpu
@pytest.mark.parametrize("H,W,expect", [(4095, 4096, "tc128"), (4096, 4096, "simt")])
def test_bf16_largest_image_of_the_tensor_core_path(vb, H, W, expect):
    """The 16-bit kernel addresses corners of one channels-last image with 32-bit byte offsets, so it takes images of
    H * W * c_in < 2^30 elements; 4095 x 4096 x 64 is just under, 4096 x 4096 x 64 the first shape over (SIMT).  A 1x1
    kernel with random offsets samples the whole image; the last row, the last column and the second image are checked."""
    from vision_b200 import _lib

    B, C, Co = 2, 64, 128
    ws = _lib.core().vb200_deform_conv2d_workspace_bytes(CODE[torch.bfloat16], B, C, H, W, Co, 1, 1, H, W, 1, 1)
    assert ("simt" if ws == 0 else "tc") == path_class(expect)
    gen = torch.Generator(device=DEV).manual_seed(H)
    x = torch.randn(B, C, H, W, device=DEV, dtype=torch.bfloat16, generator=gen)
    off = (torch.randn(B, 2, H, W, device=DEV, generator=gen) * 3).to(torch.bfloat16)
    off[:, :, -1, -1] = 0                                    # the very last pixel of each image, exactly
    off[:, :, -2, -2] = 1
    off[1, :, -1, :64] = 0.5
    m = torch.randn(B, 1, H, W, device=DEV, generator=gen).to(torch.bfloat16)
    w = (torch.randn(Co, C, 1, 1, device=DEV, generator=gen) / 8).to(torch.bfloat16)
    b = torch.randn(Co, device=DEV, generator=gen).to(torch.bfloat16)
    got, kernels = launched_forward_kernels(lambda: vb.ops.deform_conv2d(x, off, w, b, 1, 0, 1, m))
    assert kernels == {expect}, kernels
    last_row = (H - 1) * W + torch.arange(0, W, 37, device=DEV)
    last_col = torch.arange(0, H, 29, device=DEV) * W + W - 1
    rnd = torch.randint(0, H * W, (256,), device=DEV, generator=gen)
    pix = torch.cat([last_row, last_col, rnd, torch.tensor([0, W - 1, (H - 1) * W, H * W - 1, H * W - W - 2], device=DEV)])
    ref = dcn_ref64(x, off, w, b, (1, 1), (0, 0), (1, 1), m, pixels=pix)
    r = worst_ratio(got.flatten(2)[:, :, pix], ref, F16_BOUND)
    print(f"{H}x{W}x{C} bf16 [{expect}] worst ratio {r:.3g}")
    assert r <= 1, f"worst ratio {r:.3g}"


# =============================== GPU: large kernels through torchvision ===============================
@pytest.mark.gpu
def test_torchvision_deform_conv2d_11x11_after_install(vb):
    """KK = 121 takes the SIMT kernel, whose sampling table holds at most 106 taps: it is built in chunks of taps."""
    import torchvision

    assert dcn_path(torch.float32, 16, 24, 11, 11, 1, 2) == "simt"
    gen = torch.Generator().manual_seed(11)
    x, off, w, b, m = make_inputs(gen, 2, 16, 21, 18, 24, (11, 11), (1, 1), (5, 4), (1, 1), 1, 2, dtype=torch.float32, device=DEV)
    was = vb.installed()
    vb.install()
    try:
        before = vb.launch_count()
        got, kernels = launched_forward_kernels(lambda: torchvision.ops.deform_conv2d(x, off, w, b, padding=(5, 4), mask=m))
        assert vb.launch_count() > before
        assert kernels == {"simt"}, kernels
    finally:
        if not was:
            vb.uninstall()
    r = worst_ratio(got, dcn_ref64(x, off, w, b, (1, 1), (5, 4), (1, 1), m), F32_BOUND)
    assert r <= 1, f"worst ratio {r:.3g}"
