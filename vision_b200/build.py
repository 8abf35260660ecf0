"""In-tree build of the two shared libraries (no JIT cache: the .so files travel with the repo).

  vision_b200/lib/libvision_b200.so    C-ABI CUDA kernels, nvcc -gencode arch=compute_90a,code=sm_90a
  vision_b200/lib/libvision_b200_torch.so   torch dispatcher shim (g++, links the above)

`python -m vision_b200.build [--force]`
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "build")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

CU_SOURCES = ["runtime.cu", "box_iou_rotated.cu", "roi_ops.cu", "roi_backward.cu", "nms.cu", "resize.cu", "resize_stream.cu", "deform_conv2d.cu", "deform_conv2d_bwd.cu",
              "deform_conv2d_tc.cu", "keypoints.cu", "rcnn_transform.cu", "matching.cu"]
CORE_LIB = os.path.join(LIBDIR, "libvision_b200.so")
SHIM_LIB = os.path.join(LIBDIR, "libvision_b200_torch.so")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr", "-Wno-deprecated-declarations",
              "-I", INCLUDE]


def _nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found (needed to build vision_b200)")
    return cand


def _newer(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(d) <= t for d in deps)


def build_core(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    # every header under csrc/ and include/ is a dependency of every object (struct layouts such as DcnParams and the
    # mbarrier helpers are shared between translation units; a stale object would link silently)
    import glob

    headers = sorted(glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(CSRC, "*.cuh")) +
                     glob.glob(os.path.join(INCLUDE, "*.h")))
    nvcc = _nvcc()
    objs = []

    def compile_one(src: str) -> str:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJDIR, src.replace(".cu", ".o"))
        if force or not _newer(o, [s] + headers):
            cmd = [nvcc] + NVCC_FLAGS + ["-c", s, "-o", o]
            if verbose:
                print(" ".join(cmd), flush=True)
            subprocess.check_call(cmd)
        return o

    with ThreadPoolExecutor(max_workers=min(8, len(CU_SOURCES))) as ex:
        objs = list(ex.map(compile_one, CU_SOURCES))
    if force or not _newer(CORE_LIB, objs):
        # default (static) cudart: the library carries its own runtime and attaches to the
        # primary context torch already created; streams are plain CUstream handles.
        cmd = [nvcc, "-shared", "-o", CORE_LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    return CORE_LIB


def build_shim(force: bool = False, verbose: bool = False) -> str:
    import torch
    from torch.utils import cpp_extension as ce

    src = os.path.join(CSRC, "torch_shim.cpp")
    deps = [src, os.path.join(INCLUDE, "vision_b200.h"), CORE_LIB]
    if not force and _newer(SHIM_LIB, deps):
        return SHIM_LIB
    inc = []
    for p in ce.include_paths():
        inc += ["-isystem", p]
    cuda_home = os.environ.get("CUDA_HOME") or "/usr/local/cuda"
    inc += ["-isystem", os.path.join(cuda_home, "include")]
    torch_lib = os.path.join(os.path.dirname(torch.__file__), "lib")
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-DTORCH_API_INCLUDE_EXTENSION_H",
           f"-D_GLIBCXX_USE_CXX11_ABI={abi}", "-DUSE_CUDA", "-Wno-deprecated-declarations"] + inc + [
        src, "-o", SHIM_LIB, "-L", LIBDIR, "-lvision_b200", "-L", torch_lib, "-lc10", "-lc10_cuda", "-ltorch_cpu",
        "-ltorch_cuda", "-ltorch", "-Wl,-rpath,$ORIGIN", f"-Wl,-rpath,{torch_lib}", "-Wl,--no-as-needed"]
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    return SHIM_LIB


def build_all(force: bool = False, verbose: bool = False) -> tuple[str, str]:
    core = build_core(force, verbose)
    shim = build_shim(force, verbose)
    return core, shim


if __name__ == "__main__":
    f = "--force" in sys.argv
    print(build_all(force=f, verbose=True))
