"""In-tree build of libmagnet_b200.so (sm_90a, H100) with plain nvcc — no torch extension machinery.

The C-ABI library has no torch dependency, so it is compiled straight from magnet_b200/csrc/*.cu
into magnet_b200/libmagnet_b200.so (object files and logs under magnet_b200/_build/).
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
BUILD = PKG / "_build"
LIB = PKG / "libmagnet_b200.so"
SOURCES = ["api.cu", "cost_mma.cu", "cost_tma.cu", "cost_cells.cu", "cost_direct.cu", "cost_f_bwd.cu", "cost_f_bwd_mma.cu", "cost_cw_bwd.cu", "fnet_l1.cu",
           "plane_depth.cu", "aux_kernels.cu", "depth_metrics.cu", "gnet_head.cu", "mask_head.cu", "dnet_head.cu"]
HEADERS = [CSRC / "common.cuh", CSRC / "cells_common.cuh", CSRC / "tma_common.cuh", CSRC / "cw_mask.cuh",
           CSRC / "upsample_common.cuh", CSRC / "gaussian_common.cuh", CSRC / "head_common.cuh", CSRC / "soft_argmin.cuh", PKG.parent / "include" / "magnet_b200.h"]
ARCH = "arch=compute_90a,code=sm_90a"
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", ARCH, "-lineinfo",
              "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; cannot build libmagnet_b200.so")


def _digest() -> str:
    h = hashlib.sha256()
    for f in [CSRC / s for s in SOURCES] + HEADERS:
        h.update(f.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False, defines=(), tag: str = "") -> Path:
    """Compile every .cu for sm_90a and link the shared library.  No-op when up to date.
    ``defines`` / ``tag`` build a tuning variant (e.g. defines=("MAGNET_NCELL=4",), tag="nc4") into
    libmagnet_b200_<tag>.so, selectable at run time with the MAGNET_B200_LIB environment variable."""
    BUILD.mkdir(exist_ok=True)
    lib = LIB if not tag else PKG / f"libmagnet_b200_{tag}.so"
    stamp = BUILD / f"digest{tag}.txt"
    dig = _digest() + "|" + ",".join(defines)
    if not force and lib.exists() and stamp.exists() and stamp.read_text() == dig:
        return lib
    nvcc = _nvcc()

    def compile_one(src: str):
        obj = BUILD / (src + tag + ".o")
        cmd = [nvcc, *NVCC_FLAGS, *[f"-D{d}" for d in defines], "-I", str(PKG.parent / "include"), "-c",
               str(CSRC / src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        (BUILD / (src + tag + ".log")).write_text(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [nvcc, "-shared", "-gencode", ARCH, "-o", str(lib), *map(str, objs)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    stamp.write_text(dig)
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
