"""Builds libdepthmap_b200.so (the C-ABI of include/depthmap_b200.h) for sm_90a, in-tree.

    python stable-diffusion-webui-depthmap-script_b200/csrc/build.py [--force] [--verbose]

nvcc cross-compiles without a GPU.  Exact-arithmetic translation units are built with -fmad=false because the
reference's numba / numpy / OpenCV code performs no FMA contraction; tensor-core units use the default.
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
OUT_DIR = os.path.join(PKG, "_native")
OBJ_DIR = os.path.join(OUT_DIR, "obj")
LIB = os.path.join(OUT_DIR, "libdepthmap_b200.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden"]

# (source, extra flags)
UNITS = [
    ("capi_common.cu", []),
    ("normalize.cu", ["-fmad=false"]),
    ("normalmap.cu", ["-fmad=false"]),
    ("stereo.cu", ["-fmad=false"]),
]
for _extra in ("vit_kernels.cu", "gemm_wgmma.cu", "attention_wgmma.cu", "zoe_kernels.cu", "leres_kernels.cu", "midas_kernels.cu", "boost_kernels.cu", "pos_tables.cu", "png_encode.cu"):
    if os.path.exists(os.path.join(HERE, _extra)):
        UNITS.append((_extra, []))

HEADERS = [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith((".cuh", ".h"))] + \
          [os.path.join(os.path.dirname(PKG), "include", "depthmap_b200.h")]


def _newer(target, deps):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(d) <= t for d in deps if os.path.exists(d))


def build(force=False, verbose=False):
    os.makedirs(OBJ_DIR, exist_ok=True)
    nvcc = os.environ.get("NVCC", "nvcc")
    objs = []
    rebuilt = False
    for src, extra in UNITS:
        s = os.path.join(HERE, src)
        o = os.path.join(OBJ_DIR, src.replace(".cu", ".o"))
        objs.append(o)
        if not force and _newer(o, [s] + HEADERS + [os.path.abspath(__file__)]):
            continue
        cmd = [nvcc] + ARCH + COMMON + extra + ["-c", s, "-o", o]
        if verbose:
            cmd += ["-Xptxas", "-v"]
            print(" ".join(cmd))
        subprocess.run(cmd, check=True)
        rebuilt = True
    if rebuilt or not os.path.exists(LIB):
        cmd = [nvcc] + ARCH + ["-shared", "-o", LIB] + objs + ["-Xcompiler", "-fPIC"]
        if verbose:
            print(" ".join(cmd))
        subprocess.run(cmd, check=True)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
