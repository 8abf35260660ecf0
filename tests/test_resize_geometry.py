"""resize across the geometries its three kernels accept, against a float64 evaluation of the same operation.

vb200_resize runs one of three kernels: resize_aa_stream_kernel<T, NP, NW> (bilinear antialias downscale: every input
row streams once through shared memory, thread i owns the input pixels between output centres i - 1 and i and reads a
slot of 2 NP pixels of each row, NW = 8 or 16 consumer warps), resize_aa_generic_kernel (any antialias filter and scale)
and resize_noaa_kernel (antialias=False).  `stream_plan` restates the host rules that pick the kernel and the stream
kernel's launch shape (resize_aa_stream_try, dispatch_lw and launch_stream in resize_stream.cu).  Without a GPU the case
table is shown to reach all 36 stream instantiations, both band-height branches, single-band grids and every reason the
stream path declines; on the GPU every case asserts that the kernel it launched (its name in a torch.profiler trace) is
the one the plan names, so a change of the dispatch rules fails here instead of quietly shrinking the coverage.  (Late
in the whole GPU suite the profiler at times delivers no record of a kernel the library counted as launched; such a case
still runs its numeric checks and then reports itself skipped, never passed.)

Ground truth, per case: `ref64`, torch.nn.functional.interpolate on the CPU in float64 of the values the kernel reads
(the storage-type input widened exactly), and the reference's own route on the GPU: fp32 interpolate of the widened
input, then the cast torchvision applies (_geometry.py:340-360: round to nearest even for fp16 / bf16; clamp for bicubic,
round half to even and cast for uint8).  d_ref = max |route_fp32 - ref64| is the reference's own fp32 error on the case
(its weights and spans are computed in float).  Bounds, per element:
  fp32          |got - ref64| <= 1.25 d_ref + 1e-6
  fp16 / bf16   |got - ref64| <= ulp(ref64) + d_ref     (ulp of the storage type at |ref64|)
  uint8         |got - clamp(ref64)| <= 0.5 + d_ref
and for the 16-bit and uint8 outputs, got equals the route's output except where the route's fp32 value lies within
d_ref of a rounding midpoint; such disagreements stay below MAX_TIE_SHARE of the elements.

Non-finite pixels (+inf, -inf, NaN) are held to the route's output exactly: the same NaN positions, the same infinities
with the same signs; the elements finite in both to the bounds above.  The stream kernel does not meet the first part
(DESIGN.md section 8): for its cases a NonFinitePositions error, raised after every other check passed, is a strict
expected failure."""
import math
import re
import zlib
from dataclasses import dataclass
from typing import Optional

import numpy as np
import pytest
import torch
import torch.nn.functional as F

DEV = "cuda"
F16, BF16, F32, U8 = torch.float16, torch.bfloat16, torch.float32, torch.uint8
ALL = (F16, BF16, F32, U8)
FLOATS = (F16, BF16, F32)
ESIZE = {F16: 2, BF16: 2, F32: 4, U8: 1}
H100_SMS, H100_SMEM_OPTIN = 132, 232448          # multiProcessorCount, sharedMemPerBlockOptin (227 KB)
MAX_TIE_SHARE = 1e-2

# resize_stream.cu constants
K_MAX_CONSUMER_WARPS, K_MAX_BAND_ROWS = 16, 1024
NP_BUCKETS = {8: (4, 6, 10, 12, 16), 16: (4, 6, 10, 16)}
DECLINES = ("bicubic", "horizontal upscale", "vertical upscale", "too wide", "row bytes", "pointer", "scale_w < 2",
            "slot", "band", "smem")


# =============================== the dispatch rules, restated ===============================
@dataclass(frozen=True)
class Plan:
    kernel: str                            # "stream", "generic" or "noaa"
    decline: Optional[str] = None          # why an antialias bilinear request is not streamed (one of DECLINES)
    dtype: Optional[torch.dtype] = None
    np_: int = 0                           # pixel pairs per slot
    nw: int = 0                            # consumer warps compiled for
    splits: int = 0                        # CTAs along the output rows of a plane
    rows_out_per_cta: int = 0
    resplit: bool = False                  # band taller than kMaxBandRows: rows_out_per_cta cut to fit

    def label(self):
        return ("stream", self.dtype, self.np_, self.nw) if self.kernel == "stream" else (self.kernel,)


def ceil_div(a, b):
    return (a + b - 1) // b


def stream_plan(dtype, planes, in_h, in_w, out_h, out_w, mode="bilinear", antialias=True, aligned=True, sms=H100_SMS,
                smem_optin=H100_SMEM_OPTIN):
    """The kernel vb200_resize launches for these arguments (aligned: the input pointer is 16-byte aligned).  Float
    arithmetic is fp32 where the host code's is."""
    if not antialias:
        return Plan("noaa")
    generic = lambda why: Plan("generic", decline=why)
    if mode != "bilinear":
        return generic("bicubic")
    es = ESIZE[dtype]
    if in_w <= out_w:
        return generic("horizontal upscale")
    if in_h < out_h:
        return generic("vertical upscale")
    if out_w + 1 > 31 * K_MAX_CONSUMER_WARPS:
        return generic("too wide")
    if in_w * es % 16:
        return generic("row bytes")
    if not aligned:
        return generic("pointer")
    scale_w, scale_h = np.float32(in_w) / np.float32(out_w), np.float32(in_h) / np.float32(out_h)
    if scale_w < np.float32(2):
        return generic("scale_w < 2")
    # dispatch_lw: a thread owns at most floor(scale) + 1 pixels, plus the slot's alignment slack
    align = 4 if es == 1 else 2
    need = (int(np.floor(scale_w)) + 1 + (align - 1) + 1) // 2
    nw = 8 if ceil_div(out_w + 1, 31) <= 8 else K_MAX_CONSUMER_WARPS
    np_ = next((b for b in NP_BUCKETS[nw] if need <= b), None)
    if np_ is None:
        return generic("slot")
    # launch_stream
    lw = (np_ * 2 * es + 3) // 4
    row_pitch = (in_w * es + lw * 4 + 4 + 127) & ~127
    splits = ceil_div(sms * 3 * 2, planes)
    splits = max(1, min(splits, out_h))
    if splits > 1 and out_h // splits < 8:
        splits = out_h // 8 if out_h // 8 > 0 else 1
    rows = ceil_div(out_h, splits)
    splits = ceil_div(out_h, rows)
    band_rows = int(np.float32(rows + 2) * scale_h) + 4
    resplit = band_rows > K_MAX_BAND_ROWS
    if resplit:
        rows = int(np.float32(K_MAX_BAND_ROWS - 4) / scale_h) - 2
        if rows < 1:
            return generic("band")
        splits = ceil_div(out_h, rows)
        band_rows = int(np.float32(rows + 2) * scale_h) + 4
    band_cap = (band_rows + 31) & ~31
    fixed = (out_w + out_h) * 16 + band_cap * 12 + 256
    ctas_per_sm = 3 if nw <= 8 and np_ <= 12 else 2
    budget = (smem_optin - 3072) // ctas_per_sm - 1024
    if budget < fixed + 3 * row_pitch:
        return generic("smem")
    return Plan("stream", dtype=dtype, np_=np_, nw=nw, splits=splits, rows_out_per_cta=rows, resplit=resplit)


# =============================== the case table ===============================
@dataclass(frozen=True)
class Case:
    planes: int
    in_hw: tuple
    out_hw: tuple
    mode: str = "bilinear"
    aa: bool = True
    dtypes: tuple = ALL
    aligned: bool = True                   # False: the input starts one element past a 16-byte boundary

    def plan(self, dtype, **dev):
        return stream_plan(dtype, self.planes, *self.in_hw, *self.out_hw, mode=self.mode, antialias=self.aa,
                           aligned=self.aligned, **dev)


# Widths are multiples of 16 unless a case says otherwise, so that the row-alignment rule lets every storage type stream;
# the types then differ in slot alignment (2 pixels for 16- and 32-bit types, 4 for uint8) and so in NP.  "fN" names
# floor(scale_w) = N, the top of an NP bucket for one of the two alignments (the slot is then as full as it gets).
CASES = {
    # 8 consumer warps (out_w <= 247): NP 4 / 6 / 10 / 12 / 16 for both slot alignments; f30 is past uint8's largest slot
    "w37_f4": Case(3, (45, 176), (11, 37)),
    "w37_f6": Case(3, (45, 256), (11, 37)),
    "w37_f8": Case(3, (45, 320), (11, 37)),
    "w37_f10": Case(3, (45, 400), (11, 37)),
    "w37_f16": Case(3, (45, 624), (11, 37)),
    "w37_f18": Case(3, (45, 688), (11, 37)),
    "w37_f20": Case(3, (45, 768), (11, 37)),
    "w37_f22": Case(3, (45, 848), (11, 37)),
    "w37_f28": Case(3, (45, 1072), (11, 37)),
    "w37_f30": Case(3, (45, 1136), (11, 37)),
    "w247_f2": Case(2, (40, 736), (17, 247)),                 # the widest output on 8 warps
    # 16 consumer warps (248 <= out_w <= 495); fp32 rows of 14352 pixels leave no room for three stages
    "w248_f4": Case(2, (12, 1232), (6, 248)),                 # the narrowest output on 16 warps
    "w263_f8": Case(2, (12, 2352), (5, 263)),
    "w300_f16": Case(2, (10, 5088), (4, 300)),
    "w300_f20": Case(2, (8, 6288), (4, 300)),                 # no NP 12 on 16 warps: NP 16
    "w495_f28": Case(2, (6, 14352), (3, 495)),                # the widest output the stream kernel takes
    "w496": Case(2, (8, 992), (4, 496)),                      # one column too wide: generic
    # one output column: two intervals, lane 0 the only writer (its output needs lane 1's partial), interval 1 ends at
    # in_w; the generic kernel's one-column tile; the gather's clamp at both edges
    "w1": Case(3, (40, 16), (10, 1)),
    "w1_bicubic": Case(3, (40, 16), (10, 1), mode="bicubic"),
    "w1_noaa": Case(3, (40, 16), (10, 1), aa=False),
    "w20_f40": Case(2, (40, 800), (10, 20)),                  # past every slot: generic
    # scale_w exactly 2 (NP 4: an 8-pixel slot over 2-pixel intervals) and just below it
    "scale2": Case(3, (96, 128), (48, 64)),
    "scale_below2": Case(3, (64, 128), (32, 65)),
    # vertical scale 1 (streams) and a vertical upscale (declines)
    "same_h": Case(2, (40, 640), (40, 64)),
    "up_h": Case(2, (30, 640), (45, 64)),
    # tall planes: the band of 8 output rows would exceed kMaxBandRows and is cut to 2 rows; at scale_h 350 not even
    # one output row fits a band
    "tall_resplit": Case(2, (4000, 480), (16, 24)),
    "tall_band_decline": Case(1, (3500, 64), (10, 16)),
    # 800 planes: one band per plane (splits == 1) although out_h = 16 would otherwise be cut in two
    "planes800": Case(800, (64, 128), (16, 32)),
    # more planes than a grid dimension takes: the chunk loops of all three kernels
    "planes65600": Case(65600, (8, 16), (4, 8)),
    "planes65600_bicubic": Case(65600, (8, 16), (4, 8), mode="bicubic", dtypes=(F16, U8)),
    "planes65600_noaa": Case(65600, (8, 16), (4, 8), aa=False, dtypes=(F16, U8)),
    # the input one element past an aligned address; rows of 200 bytes (16-bit) / 100 bytes (uint8), 400 for fp32
    "misaligned": Case(3, (45, 640), (11, 37), aligned=False),
    "row_not16": Case(3, (45, 100), (11, 25)),
    # the cfg5 geometry at two planes (NP 10 for the 2-pixel alignment, 12 for uint8)
    "cfg5_2planes": Case(2, (2160, 3840), (224, 224)),
    # bicubic antialias down and up, bilinear antialias up (generic)
    "bicubic_aa_down": Case(3, (90, 160), (23, 41), mode="bicubic"),
    "bicubic_aa_up": Case(3, (20, 30), (47, 71), mode="bicubic"),
    "bilinear_aa_up": Case(3, (24, 40), (50, 77)),
    # antialias=False, bilinear and bicubic, down and up (uint8 bicubic: the clamp)
    "noaa_bilinear_down": Case(3, (90, 160), (23, 41), aa=False),
    "noaa_bilinear_up": Case(3, (20, 30), (47, 71), aa=False),
    "noaa_bicubic_down": Case(3, (90, 160), (23, 41), mode="bicubic", aa=False),
    "noaa_bicubic_up": Case(3, (20, 30), (47, 71), mode="bicubic", aa=False),
}


def all_plans(**dev):
    return {(name, dt): c.plan(dt, **dev) for name, c in CASES.items() for dt in c.dtypes}


# =============================== CPU: what the table reaches ===============================
def test_case_table_reaches_every_stream_kernel_and_every_decline():
    plans = all_plans()
    stream = [p for p in plans.values() if p.kernel == "stream"]
    reached = {(p.dtype, p.np_, p.nw) for p in stream}
    every = {(dt, np_, nw) for dt in ALL for nw, nps in NP_BUCKETS.items() for np_ in nps}
    assert len(every) == 36
    assert reached == every, f"not reached: {sorted(every - reached, key=str)}"
    assert {p.resplit for p in stream} == {False, True}
    # single-band grids from the plane count alone (out_h >= 16 would otherwise be split)
    assert any(p.splits == 1 and CASES[name].out_hw[0] >= 16 for (name, _), p in plans.items() if p.kernel == "stream")
    assert any(p.splits > 1 for p in stream)
    assert {p.decline for p in plans.values() if p.kernel == "generic"} == set(DECLINES)
    assert any(p.kernel == "noaa" for p in plans.values())
    # a single output column on each kernel
    assert {p.kernel for (name, _), p in plans.items() if CASES[name].out_hw[1] == 1} == {"stream", "generic", "noaa"}


def test_stream_plan_spot_values():
    """Hand-derived plans: cfg5 at its benchmarked batch (384 planes) and at 2 planes, the tall re-split."""
    p = stream_plan(F16, 384, 2160, 3840, 224, 224)
    assert (p.kernel, p.np_, p.nw, p.splits, p.rows_out_per_cta, p.resplit) == ("stream", 10, 8, 3, 75, False)
    p = stream_plan(U8, 384, 2160, 3840, 224, 224)
    assert (p.np_, p.nw) == (12, 8)
    p = stream_plan(F16, 2, 2160, 3840, 224, 224)
    assert (p.splits, p.rows_out_per_cta, p.resplit) == (28, 8, False)
    p = stream_plan(F16, 2, 4000, 480, 16, 24)                 # 8 rows -> band 2504 > 1024 -> int(1020 / 250) - 2 = 2 rows
    assert (p.np_, p.nw, p.splits, p.rows_out_per_cta, p.resplit) == (12, 8, 8, 2, True)
    assert stream_plan(F16, 1, 3500, 64, 10, 16).decline == "band"
    assert stream_plan(F32, 2, 6, 14352, 3, 495).decline == "smem"
    assert stream_plan(F16, 2, 6, 14352, 3, 495).np_ == 16
    assert stream_plan(F16, 3, 45, 640, 11, 37, aligned=False).decline == "pointer"


def separable_aa64(x, out_hw, mode):
    """The antialias resize of x [planes, H, W] written out in float64: per axis, output i takes the inputs of its span
    [int(c - support + 0.5), int(c + support + 0.5)) around c = scale (i + 0.5), clipped to the image, weighted by the
    filter at (j + 0.5 - c) / scale and normalised by their sum (UpSample.cuh:303-343)."""
    def filt(t):
        t = abs(t)
        if mode == "bilinear":
            return max(0.0, 1.0 - t)
        a = -0.5
        return ((a + 2) * t - (a + 3)) * t * t + 1 if t < 1 else (((t - 5) * t + 8) * t - 4) * a if t < 2 else 0.0

    def axis(n_in, n_out):
        scale = n_in / n_out
        support = (1.0 if mode == "bilinear" else 2.0) * max(scale, 1.0)
        w = torch.zeros(n_out, n_in, dtype=torch.float64)
        for i in range(n_out):
            c = scale * (i + 0.5)
            for j in range(max(int(c - support + 0.5), 0), min(int(c + support + 0.5), n_in)):
                w[i, j] = filt((j + 0.5 - c) / max(scale, 1.0))
            w[i] /= w[i].sum()
        return w

    return torch.einsum("oy,pyx,wx->pow", axis(x.shape[-2], out_hw[0]), x.double(), axis(x.shape[-1], out_hw[1]))


@pytest.mark.parametrize("mode", ["bilinear", "bicubic"])
@pytest.mark.parametrize("in_hw,out_hw", [((40, 16), (10, 1)), ((16, 40), (1, 10)), ((45, 176), (11, 37)), ((20, 30), (47, 71)),
                                          ((40, 16), (1, 1))])
def test_ref64_is_the_separable_filter(mode, in_hw, out_hw):
    """The float64 reference against the filter written out, including a single output column."""
    x = torch.randn(3, *in_hw, generator=torch.Generator().manual_seed(sum(in_hw)), dtype=torch.float64)
    ref = interpolate_cpu(x, out_hw, mode, True)
    torch.testing.assert_close(ref, separable_aa64(x, out_hw, mode), rtol=0, atol=1e-12)


# =============================== GPU helpers ===============================
def launched_resize_kernels(fn):
    """Runs fn under torch.profiler: (its result, the plan labels of the resize kernels the trace names).

    fn is deterministic: a session whose trace names no resize kernel runs it again, up to three times."""
    from torch.profiler import ProfilerActivity, profile

    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        labels = resize_kernel_labels({e.name for e in prof.events()})
        if labels:
            break
    return out, labels


TYPE_NAMES = {"__half": F16, "6__half": F16, "__nv_bfloat16": BF16, "13__nv_bfloat16": BF16, "float": F32, "f": F32,
              "unsigned char": U8, "h": U8}


def resize_kernel_labels(names):
    """Plan labels of the resize kernels among profiled event names (demangled or mangled)."""
    labels = set()
    for n in names:
        m = re.search(r"resize_aa_stream_kernel<([^,]+), (\d+), (\d+)>", n) or re.search(r"resize_aa_stream_kernelI(\w+?)Li(\d+)ELi(\d+)E", n)
        if m:
            labels.add(("stream", TYPE_NAMES[m.group(1).strip()], int(m.group(2)), int(m.group(3))))
        elif "resize_aa_generic_kernel" in n:
            labels.add(("generic",))
        elif "resize_noaa_kernel" in n:
            labels.add(("noaa",))
    return labels


def device_limits():
    props = torch.cuda.get_device_properties(0)
    return dict(sms=props.multi_processor_count, smem_optin=props.shared_memory_per_block_optin)


def make_input(case, dtype, seed):
    gen = torch.Generator().manual_seed(seed)
    shape = (case.planes, *case.in_hw)
    if dtype == U8:
        return torch.randint(0, 256, shape, generator=gen, dtype=torch.uint8)
    return torch.randn(shape, generator=gen).to(dtype)


def to_device(x, aligned=True):
    if aligned:
        return x.to(DEV)
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device=DEV)
    xd = buf[1:].view(x.shape)
    xd.copy_(x)
    assert xd.is_contiguous() and xd.data_ptr() % 16 != 0
    return xd


def storage_ulp(ref, dtype):
    """ulp of the 16-bit storage type at |ref| (float64), subnormals included."""
    mant, emin = {F16: (10, -14), BF16: (7, -126)}[dtype]
    e = torch.frexp(ref.abs())[1] - 1
    e = torch.where(ref == 0, torch.full_like(e, emin), e).clamp(min=emin)
    return torch.ldexp(torch.ones_like(ref), e - mant)


def route_cast(r32, dtype, mode):
    """_geometry.py:352-359, after the fp32 interpolate."""
    if dtype == U8:
        if mode == "bicubic":
            r32 = r32.clamp(0, 255)
        return r32.round().to(U8)
    return r32.to(dtype)


def interpolate_cpu(x, out_hw, mode, aa):
    """torch's CPU interpolate of x [planes, H, W] (align_corners=False).  Its antialias kernel, at an output width of 1
    under a taller output, reads the first output row's vertical span for every output row; the transposed image
    (output height 1) does not take that path, so such shapes are evaluated transposed."""
    kw = dict(mode=mode, antialias=aa, align_corners=False)
    if aa and out_hw[1] == 1 and out_hw[0] > 1:
        return F.interpolate(x.transpose(-1, -2)[None], size=[out_hw[1], out_hw[0]], **kw)[0].transpose(-1, -2)
    return F.interpolate(x[None], size=list(out_hw), **kw)[0]


def references(x, out_hw, mode, aa):
    """(ref64 on the CPU, the route's fp32 value, the route's output), the last two from torch's CUDA kernels.  torch's
    CUDA antialias kernel holds a whole filter per output in shared memory and refuses the tall cases (scale_h >= 250);
    for those the route is torch's CPU kernel."""
    kw = dict(size=list(out_hw), mode=mode, antialias=aa, align_corners=False)
    ref64 = interpolate_cpu(x.double(), out_hw, mode, aa)
    try:
        r32 = F.interpolate(x.to(DEV).float()[None], **kw)[0].cpu()
    except RuntimeError as e:
        if "shared memory" not in str(e):
            raise
        r32 = interpolate_cpu(x.float(), out_hw, mode, aa)
    return ref64, r32, route_cast(r32, x.dtype, mode)


def check_bounds(got, x, out_hw, mode, aa, label, where=None):
    """Asserts the bounds of the module docstring on the elements that are finite in ref64 and in the route (and, given
    `where`, true there)."""
    dtype = x.dtype
    ref64, r32, route = references(x.cpu(), out_hw, mode, aa)
    g = got.cpu()
    ok = torch.isfinite(ref64) & torch.isfinite(r32)
    if where is not None:
        ok &= where
    if dtype == U8:
        ref64 = ref64.clamp(0, 255)
        r32c = r32.double().clamp(0, 255)
    else:
        r32c = r32.double()
    d_ref = (r32c - ref64).abs()[ok].max().item() if ok.any() else 0.0
    err = (g.double() - ref64).abs()
    if dtype == F32:
        bound = torch.full_like(ref64, 1.25 * d_ref + 1e-6)
    elif dtype == U8:
        bound = torch.full_like(ref64, 0.5 + d_ref)
    else:
        bound = storage_ulp(ref64, dtype) + d_ref
    ratio = (err / bound)[ok].max().item() if ok.any() else 0.0
    share = 0.0
    if dtype != F32:
        d = torch.tensor(d_ref, dtype=torch.float32)
        near_tie = route_cast(r32 - d, dtype, mode) != route_cast(r32 + d, dtype, mode)
        differ = (g != route) & ok
        share = differ.double().mean().item()
        far = differ & ~near_tie
        assert not far.any(), (f"{label}: {int(far.sum())} outputs differ from the reference's route away from a rounding tie, "
                               f"e.g. got {g[far][:4].tolist()} route {route[far][:4].tolist()} fp32 {r32[far][:4].tolist()}")
    print(f"RESIZE {label} d_ref={d_ref:.3g} worst |got-ref64|/bound={ratio:.3g} tie-share={share:.2e}")
    assert ratio <= 1, f"{label}: worst |got - ref64| / bound = {ratio:.3g} (d_ref {d_ref:.3g})"
    assert share <= MAX_TIE_SHARE, f"{label}: {share:.3g} of the outputs differ from the route at rounding ties"


def run_resize(vb, x_cpu, case, dtype):
    """Resizes x_cpu on the GPU under the profiler: (output on the GPU, the launched kernel's plan label, the plan)."""
    xd = to_device(x_cpu, case.aligned)
    plan = case.plan(dtype, **device_limits())
    before = vb.launch_count()
    got, labels = launched_resize_kernels(
        lambda: vb.transforms.resize_image(xd, list(case.out_hw), interpolation=case.mode, antialias=case.aa))
    assert vb.launch_count() > before, "no vision_b200 kernel ran"
    assert got.shape == (case.planes, *case.out_hw) and got.dtype == dtype
    return got, labels, plan


def check_kernel(labels, plan, label):
    """True when the trace named the planned kernel; an assertion error when it named another.  An empty set (the
    profiler delivered no record of a kernel the library counted as launched, see run_resize) is not a verdict: the
    caller skips after its numeric checks."""
    assert not labels or labels == {plan.label()}, f"{label}: the plan names {plan.label()}, launched {labels}"
    return bool(labels)


NO_RECORD = ("the profiler delivered no record of the kernel the library counted as launched; the numeric checks ran, the "
             "kernel-name check did not")


def kernel_name(plan):
    return {"stream": f"stream<{str(plan.dtype)[6:]}, {plan.np_}, {plan.nw}>", "generic": "generic", "noaa": "noaa"}[plan.kernel]


# =============================== GPU: geometry matrix ===============================
@pytest.mark.gpu
@pytest.mark.parametrize("name,dtype", [(n, dt) for n, c in CASES.items() for dt in c.dtypes],
                         ids=[f"{n}-{str(dt)[6:]}" for n, c in CASES.items() for dt in c.dtypes])
def test_resize_matrix(vb, name, dtype):
    case = CASES[name]
    x = make_input(case, dtype, zlib.crc32(f"{name}/{dtype}".encode()) % 100_000)
    got, labels, plan = run_resize(vb, x, case, dtype)
    named = check_kernel(labels, plan, name)
    check_bounds(got, x, case.out_hw, case.mode, case.aa, f"{kernel_name(plan)}/{name}")
    if not named:
        pytest.skip(NO_RECORD)


# =============================== GPU: non-finite pixels ===============================
NONFINITE = {
    "stream_np4_scale2": Case(4, (32, 64), (16, 32), dtypes=FLOATS),          # 8-pixel slot over 2-pixel intervals
    "stream_np10": Case(4, (45, 624), (11, 37), dtypes=FLOATS),
    "stream_nw16": Case(4, (12, 1232), (6, 248), dtypes=FLOATS),
    "generic_bicubic": Case(4, (40, 90), (17, 23), mode="bicubic", dtypes=FLOATS),
    "generic_bilinear_up": Case(4, (20, 30), (47, 71), dtypes=FLOATS),
    "noaa_bilinear": Case(4, (40, 90), (17, 45), aa=False, dtypes=FLOATS),            # scale 2: samples both edge columns
    "noaa_bicubic_up": Case(4, (20, 30), (47, 71), mode="bicubic", aa=False, dtypes=FLOATS),
}
PATTERNS = ("pixels", "rows_cols", "edges")


def scatter_non_finite(x, pattern, gen):
    """Writes +inf, -inf and NaN into a copy of x (planes, H, W) by pattern: "pixels" (single pixels), "rows_cols"
    (whole rows and whole columns), "edges" (the first and the last column, where slots are clamped and padded)."""
    x = x.clone()
    P, H, W = x.shape
    vals = (math.inf, -math.inf, math.nan)
    if pattern == "pixels":
        for p in range(P):
            for k in range(3):
                x[p, torch.randint(0, H, (1,), generator=gen), torch.randint(0, W, (1,), generator=gen)] = vals[(p + k) % 3]
    elif pattern == "rows_cols":
        for p in range(P - 1):
            r, c = int(torch.randint(0, H, (1,), generator=gen)), int(torch.randint(0, W, (1,), generator=gen))
            x[p, r, :] = vals[p % 3]
            x[p + 1, :, c] = vals[(p + 1) % 3]
    else:
        x[0, :, 0] = math.inf
        x[1, :, W - 1] = math.nan
        x[2, :, 0], x[2, :, W - 1] = -math.inf, math.inf
        x[3, H // 2, 0], x[3, H // 3, W - 1] = math.nan, -math.inf
    return x


class NonFinitePositions(AssertionError):
    """Outputs whose NaN / +-inf status differs from the reference route's."""


STREAM_NON_FINITE = pytest.mark.xfail(strict=True, raises=NonFinitePositions, reason=(
    "resize_aa_stream_kernel multiplies the slot pixels outside a thread's interval by weight 0, so an inf / NaN there is "
    "NaN in that thread's outputs (DESIGN.md section 8); whole rows of inf reach every slot wider than its interval"))


@pytest.mark.gpu
@pytest.mark.parametrize("name,dtype", [pytest.param(n, dt, id=f"{n}-{str(dt)[6:]}", marks=STREAM_NON_FINITE if n.startswith("stream") else ())
                                        for n, c in NONFINITE.items() for dt in c.dtypes])
def test_non_finite_pixels_match_the_reference_route(vb, name, dtype):
    """Every pattern runs the kernel-name check and the bounds on the elements finite in both outputs first; differing
    NaN / inf positions are raised last, as NonFinitePositions, so the stream cases' expected failure covers them only."""
    case = NONFINITE[name]
    named, differ = True, []
    for pattern in PATTERNS:
        label = f"{name}-{pattern}"
        seed = zlib.crc32(f"{name}/{dtype}/{pattern}".encode()) % 100_000
        x = scatter_non_finite(make_input(case, F32, seed).to(dtype), pattern, torch.Generator().manual_seed(seed))
        got, labels, plan = run_resize(vb, x, case, dtype)
        assert plan.kernel == name.split("_")[0], plan
        named = check_kernel(labels, plan, label) and named
        _, _, route = references(x, case.out_hw, case.mode, case.aa)
        g = got.cpu()
        assert not torch.isfinite(route).all() and torch.isfinite(route).any()
        check_bounds(got, x, case.out_hw, case.mode, case.aa, f"{kernel_name(plan)}/nonfinite-{label}",
                     where=torch.isfinite(g) & torch.isfinite(route))
        nan_g, nan_r = g.isnan(), route.isnan()
        if not torch.equal(nan_g, nan_r):
            differ.append(f"{label}: NaN at {int((nan_g & ~nan_r).sum())} outputs the route has not, missing at "
                          f"{int((nan_r & ~nan_g).sum())}")
        for sign in (1, -1):
            inf_g, inf_r = g == sign * math.inf, route == sign * math.inf
            if not torch.equal(inf_g, inf_r):
                differ.append(f"{label}: {'+' if sign > 0 else '-'}inf at {int((inf_g & ~inf_r).sum())} outputs the route "
                              f"has not, missing at {int((inf_r & ~inf_g).sum())}")
    if differ:
        raise NonFinitePositions("; ".join(differ))
    if not named:
        pytest.skip(NO_RECORD)
