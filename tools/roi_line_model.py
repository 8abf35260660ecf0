"""Cost model of roi_align's line kernel (roi_align_line_kernel in vision_b200/csrc/roi_ops.cu) at the cfg2 workload.

    python tools/roi_line_model.py [--no-sass] [--k 1000] [--seed 0]

Per (RoI, plane) item it predicts, averaged over the RoIs of workloads.cfg2_roi_align:
  * tap wavefronts: the 28 tap LDS (14 loop-axis samples x their two taps) of one item.  A wavefront count of one LDS is
    the largest number of DISTINCT words any one of the 32 banks is asked for - the rule of bank_multiplicity() in the
    geometry kernel.  Lanes past the 28 taps repeat lane 0's address (a broadcast, never an extra wavefront);
  * loop-entry wavefronts: 7 warp-uniform LDS.128 of the 14 (offset, weight) loop entries, 2 wavefronts each;
  * their total.
for each lane arrangement:
  * x / y / best-of-x-y: the lane axis fixed to x, fixed to y, or chosen per RoI by the geometry kernel's rule (fewer
    conflicts on one line) - the last one is what the kernel runs;
  * half-line: the lane axis's 7 bins split into bins 0-3 (lanes 0-15) and 4-6 (lanes 16-27); group B reads the line one
    loop-axis bin further on (modulo 7), so the 28 LDS still cover every (lane tap, loop tap) pair once; chosen per RoI
    among the four (axis, half) combinations by the fewest predicted wavefronts.
The geometry is the kernel's fp32 arithmetic (roi_geometry / sample_coord / axis_entry / packed_axis in
roi_geometry.cuh), evaluated in numpy float32 one rounding per operation.

Unless --no-sass, it also compiles roi_ops.cu for sm_90a (nvcc -O3 -Xptxas -v), prints the registers / stack / spills of
each line-kernel instantiation, and counts the SASS instructions of the per-item loop (from the loop's head to its backward
branch) by opcode class; ROI_OPS_CU=<path> counts another version of the file (e.g. a parent commit's).  These are
predictions and static counts; only a GPU run gives times.
"""
from __future__ import annotations

import argparse
import collections
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

P, SR = 7, 2
NS, NL = P * SR, P * SR * 2            # loop-axis samples, lanes carrying a tap
f32 = np.float32


# ---- geometry (roi_geometry.cuh, fp32, aligned=False) ---------------------------------------------------------------
def line_pitch(w: int) -> int:
    return (w + 2) | 1


def sample_coords(start, bin_, n):
    """sample_coord for samples 0..n-1 of P bins: (start + p * bin) + ((i + .5) * bin) / SR, each op rounded to fp32"""
    j = np.arange(n)
    p, i = (j // SR).astype(f32), (j % SR).astype(f32)
    a = (start[:, None] + (p[None, :] * bin_[:, None]).astype(f32)).astype(f32)
    b = (((i + f32(0.5)).astype(f32)[None, :] * bin_[:, None]).astype(f32) / f32(SR)).astype(f32)
    return (a + b).astype(f32)


def packed_axis(v, size):
    """axis_entry + packed_axis: the low tap index of each sample (size - 2 at the border, size when outside)"""
    out = (v < -1) | (v > size)
    v = np.where(v <= 0, f32(0), v)
    lo = v.astype(np.int64)                       # (int)v truncates toward zero; v >= 0 here
    lo = np.where(lo >= size - 1, size - 2, lo)
    return np.where(out, size, lo)


def roi_geometry(rois, scale, H, W):
    r = rois.astype(f32)
    sc = f32(scale)
    sw, sh = (r[:, 1] * sc).astype(f32), (r[:, 2] * sc).astype(f32)
    ew, eh = (r[:, 3] * sc).astype(f32), (r[:, 4] * sc).astype(f32)
    rw, rh = np.maximum((ew - sw).astype(f32), f32(1)), np.maximum((eh - sh).astype(f32), f32(1))
    bw, bh = (rw / f32(P)).astype(f32), (rh / f32(P)).astype(f32)
    return packed_axis(sample_coords(sw, bw, NS), W), packed_axis(sample_coords(sh, bh, NS), H)


# ---- bank model ---------------------------------------------------------------------------------------------------
def wavefronts(addr):
    """addr [N, 32] word addresses of one LDS per row -> per row, the largest count of distinct words asked of one bank"""
    a = np.sort(addr, axis=-1)
    distinct = np.concatenate([np.ones((a.shape[0], 1), bool), a[:, 1:] != a[:, :-1]], axis=-1)
    counts = np.zeros(a.shape[0] * 32, np.int64)
    np.add.at(counts, (np.arange(a.shape[0])[:, None] * 32 + a % 32)[distinct], 1)
    return counts.reshape(-1, 32).max(axis=-1)


def lane_words(lo_lane, nb_lane):
    """word offset of each of the 32 lanes along the lane axis: lane 2j + c = tap c of sample j; lanes >= NL repeat lane 0"""
    j = np.minimum(np.arange(32) // 2, NS - 1)
    c = np.arange(32) % 2
    w = (lo_lane[:, j] + c[None, :]) * nb_lane
    w[:, NL:] = w[:, :1]
    return w


def tap_wavefronts(lane_w, loop_w, nb_loop, half: bool):
    """per RoI: wavefronts of its 28 tap LDS.  loop_w [K, NS] loop-axis word offsets of the low taps"""
    K = lane_w.shape[0]
    grp_b = np.zeros(32, bool)
    grp_b[16:NL] = True                         # lanes of lane-axis bins 4..6
    total = np.zeros(K, np.int64)
    for s in range(NS):
        s_b = (s + SR) % NS if half else s      # group B: one loop-axis bin further on, modulo the 7 bins
        off = np.where(grp_b[None, :], loop_w[:, s_b:s_b + 1], loop_w[:, s:s + 1])
        for t in (0, 1):
            total += wavefronts(lane_w + off + t * nb_loop)
    return total


def lane_axis_is_y(rois, scale, H, W):
    """per RoI, the geometry kernel's choice: lanes along y when one y line has strictly fewer conflicts than one x line"""
    pitch = line_pitch(W)
    xlo, ylo = roi_geometry(rois, scale, H, W)
    return wavefronts(lane_words(ylo, pitch)) < wavefronts(lane_words(xlo, 1))


def model(rois, scale, H, W):
    pitch = line_pitch(W)
    xlo, ylo = roi_geometry(rois, scale, H, W)
    lanes = {"x": (lane_words(xlo, 1), ylo * pitch, pitch), "y": (lane_words(ylo, pitch), xlo, 1)}
    taps = {}
    for axis, (lw, loop_w, nb) in lanes.items():
        taps[axis] = tap_wavefronts(lw, loop_w, nb, False)
        taps[axis + "/half"] = tap_wavefronts(lw, loop_w, nb, True)
    pick_y = lane_axis_is_y(rois, scale, H, W)
    taps["best-of-x-y"] = np.where(pick_y, taps["y"], taps["x"])
    four = np.stack([taps["x"], taps["y"], taps["x/half"], taps["y/half"]])
    choice = four.argmin(axis=0)
    taps["half-line"] = four.min(axis=0)
    share = {name: float((choice == i).mean()) for i, name in enumerate(["x", "y", "x/half", "y/half"])}
    ext_x = (xlo.max(1) - xlo.min(1) + 2)
    ext_y = (ylo.max(1) - ylo.min(1) + 2)
    return taps, share, float(((ext_x > 32) & (ext_y > 32)).mean()), float(pick_y.mean())


# ---- SASS ---------------------------------------------------------------------------------------------------------
CLASSES = [("LDS.128", r"^LDS\.128\b"), ("LDS", r"^LDS\b"), ("SHFL", r"^SHFL"), ("LDGSTS", r"^LDGSTS"), ("LDG", r"^LDG\."),
           ("STG/ST", r"^(STG|ST|RED)\b"), ("FP", r"^F(ADD|MUL|FMA|SEL)"), ("IMAD", r"^IMAD"),
           ("IADD3/LEA/LOP3/SHF", r"^(IADD3|LEA|LOP3|SHF|VIADD|IADD|SEL|PRMT|MOV)"), ("LDC/S2R", r"^(LDC|ULDC|S2R|S2UR)"),
           ("ISETP", r"^ISETP"), ("BRA.DIV", r"^BRA\.DIV"), ("BRA", r"^BRA\b"), ("BSSY/BSYNC", r"^(BSSY|BSYNC)"),
           ("sync", r"^(WARPSYNC|NOP|DEPBAR|LDGDEPBAR)")]


def compile_sass():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    src = os.environ.get("ROI_OPS_CU", os.path.join(ROOT, "vision_b200", "csrc", "roi_ops.cu"))
    with tempfile.TemporaryDirectory() as tmp:
        obj = os.path.join(tmp, "roi_ops.o")
        ptxas = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                                "-Wno-deprecated-declarations", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "vision_b200", "csrc"), "-Xptxas", "-v", "-c", src, "-o", obj],
                               capture_output=True, text=True, check=True).stderr
        sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return ptxas, sass


def demangle_line(name: str) -> str:
    m = re.search(r"roi_align_line_kernelILi(\d+)ELi(\d+)ELb(\d)E(?:Li(\d)E)?", name)
    return f"<{m.group(1)}, {m.group(2)}, {'MULTI' if m.group(3) == '1' else 'plain'}{', dst ' + m.group(4) if m.group(4) else ''}>" if m else name


def item_loops(sass: str):
    """per line-kernel instantiation: (name, Counter of the instructions between the item loop's head and back edge)"""
    out = []
    for block in sass.split("Function : ")[1:]:
        name = block.split("\n", 1)[0].strip()
        if "roi_align_line_kernel" not in name:
            continue
        ins = []
        for m in re.finditer(r"/\*([0-9a-f]{4,})\*/\s+(.*?);", block):
            ins.append((int(m.group(1), 16), re.sub(r"^@!?U?P\w+\s+", "", m.group(2).strip())))
        # the item loop: the backward branch whose range holds the LDS.128 of the loop entries
        best = None
        for pc, op in ins:
            mb = re.match(r"BRA\s+(?:`?\(?[\w.]*\)?)?\s*0x([0-9a-f]+)", op)
            if not mb:
                continue
            tgt = int(mb.group(1), 16)
            if tgt >= pc:
                continue
            body = [o for p, o in ins if tgt <= p <= pc]
            if sum(o.startswith("LDS.128") for o in body) >= P and (best is None or len(body) < len(best)):
                best = body
        cnt = collections.Counter()
        for o in best or []:
            mnem = o.split()[0]
            for cls, rx in CLASSES:
                if re.match(rx, mnem):
                    cnt[cls] += 1
                    break
            else:
                cnt["other"] += 1
        cnt["total"] = len(best or [])
        cnt["total w/o NOP"] = sum(1 for o in best or [] if not o.startswith("NOP"))
        out.append((name, cnt))
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=1000)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--no-sass", action="store_true")
    a = ap.parse_args()
    from vision_b200 import workloads

    x, rois, kw = workloads.cfg2_roi_align(k=a.k, seed=a.seed, channels=1)
    H, W = x.shape[-2:]
    taps, share, big, pick_y = model(rois.numpy(), kw["spatial_scale"], H, W)
    loop_entries = 7 * 2
    print(f"cfg2: {a.k} RoIs on {H}x{W} (pitch {line_pitch(W)}); {big:.0%} span > 32 feature px on both axes; "
          f"geometry kernel's lane axis today: y for {pick_y:.0%}")
    print(f"{'arrangement':<14}{'tap wf/item':>12}{'per LDS':>9}{'loop-entry wf':>15}{'total wf/item':>15}")
    for name in ("x", "y", "best-of-x-y", "x/half", "y/half", "half-line"):
        t = float(taps[name].mean())
        print(f"{name:<14}{t:12.2f}{t / 28:9.2f}{loop_entries:15d}{t + loop_entries:15.2f}")
    print("half-line choice per RoI: " + ", ".join(f"{k} {v:.0%}" for k, v in share.items()))
    if a.no_sass:
        return
    ptxas, sass = compile_sass()
    for m in re.finditer(r"Function properties for (\S*roi_align_line_kernel\S*)\n\s*(.*)\n.*Used (\d+) registers", ptxas):
        print(f"ptxas {demangle_line(m.group(1))}: {m.group(3)} registers, {m.group(2).strip()}")
    for name, cnt in item_loops(sass):
        mix = ", ".join(f"{k} {v}" for k, v in cnt.items() if k not in ("total", "total w/o NOP"))
        print(f"item loop {demangle_line(name)}: {cnt['total w/o NOP']} SASS instructions ({mix})")


if __name__ == "__main__":
    main()
