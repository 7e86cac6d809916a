"""In-tree build of libnr_b200.so (hand-written sm_90a CUDA behind the C ABI of include/nr_b200.h).

`python -m neural_renderer_b200.build [--force]` or `build_library()`; nvcc cross-compiles without a GPU.
The shared object is written next to this file (neural_renderer_b200/libnr_b200.so, git-ignored), so the package is
importable straight from the source tree.
"""
from __future__ import annotations

import os
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG_DIR)
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "libnr_b200.so")
FLAGS_PATH = LIB_PATH + ".flags"  # the nvcc flags (target architecture) the library next to it was built with
SOURCES = ["nr_api.cu", "nr_forward.cu", "nr_backward.cu", "nr_glue.cu", "nr_mip.cu", "nr_attr.cu", "nr_interior.cu", "nr_phong.cu",
           "nr_soft.cu", "nr_soft_rgb.cu", "nr_soft_uv.cu", "nr_soft_attr.cu", "nr_soft_frag.cu"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "--fmad=false",  # every fused multiply-add in this code base is an explicit __fmaf_rn (parity with the reference)
    "-Xcompiler", "-fPIC,-fvisibility=hidden",
    "-I", os.path.join(ROOT, "include"), "-I", CSRC,
]


def _sources():
    return [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def _deps():
    out = []
    for d in (CSRC, os.path.join(ROOT, "include")):
        for f in os.listdir(d):
            if f.endswith((".cu", ".cuh", ".h")):
                out.append(os.path.join(d, f))
    return out


def is_stale():
    if not os.path.exists(LIB_PATH) or not os.path.exists(FLAGS_PATH):
        return True
    with open(FLAGS_PATH) as f:
        if f.read() != " ".join(NVCC_FLAGS):
            return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(f) > t for f in _deps() if os.path.exists(f))


def build_library(force=False, verbose=False, defines=(), out=None):
    """Compile every CUDA source for sm_90a into neural_renderer_b200/libnr_b200.so (`defines` / `out`: experiment
    builds with extra -D flags into another file, selected at run time with NR_B200_LIB)."""
    if out is None and not force and not is_stale():
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "nvcc")
    objs = []
    procs = []
    build_dir = os.path.join(PKG_DIR, "build")
    os.makedirs(build_dir, exist_ok=True)
    for src in _sources():
        tag = ("." + "_".join(defines).replace("=", "-")) if defines else ""
        obj = os.path.join(build_dir, os.path.basename(src) + tag + ".o")
        cmd = [nvcc] + NVCC_FLAGS + ["-D" + d for d in defines] + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        log, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(log)
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    target = out or LIB_PATH
    cmd = [nvcc, "-shared", "-o", target] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
    subprocess.run(cmd, check=True)
    if out is None:
        with open(FLAGS_PATH, "w") as f:
            f.write(" ".join(NVCC_FLAGS))
    return target


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
