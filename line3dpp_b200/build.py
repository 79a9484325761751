"""Build libl3d_b200.so (hand-written sm_90a kernels + the C ABI) in-tree with nvcc.

    python -m line3dpp_b200.build [--force] [--verbose]

-fmad=false is part of the arithmetic contract (csrc/l3d_device.cuh): plain `a*b+c` is two IEEE roundings, fused
multiply-adds are spelled explicitly where they are wanted.
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libl3d_b200.so")
SOURCES = ["l3d_match.cu", "l3d_capi.cu", "l3d_pipeline.cu", "l3d_affinity.cu", "l3d_collinear.cu", "l3d_optimize.cu", "l3d_undistort.cu", "l3d_image_prep.cu", "l3d_jpeg.cu", "l3d_png.cu", "l3d_triangulate.cu", "l3d_pose.cu", "line3d_host.cc", "line3d_bin.cc",
           "line3d_sfm.cc", "line3d_newk.cc", "line3d_jpeg.cc", "line3d_png.cc"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-fmad=false",
         "-Xcompiler", "-fPIC,-Wno-deprecated-declarations", "-shared", "-ccbin", "/usr/bin/g++"]


def needs_build() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", h) for h in ("l3d_capi.h", "l3dpp_capi.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False, defines=(), out: str | None = None) -> str:
    """defines / out: build a variant (e.g. defines=("MK_SLOTS=4",), out="libl3d_b200_S4.so") for the geometry sweep"""
    if out is None and not force and not needs_build():
        return OUT
    target = OUT if out is None else os.path.join(HERE, out)
    cmd = [NVCC] + FLAGS + [f"-D{d}" for d in defines] + (["-Xptxas", "-v"] if verbose else []) + ["-o", target] + [os.path.join(CSRC, s) for s in SOURCES]
    if out is not None:
        subprocess.check_call(cmd)
        return target
    if verbose:
        print(" ".join(cmd))
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(OUT)
