"""Build libsinnerf_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m sinnerf_b200.build [--force] [--verbose]

The .so is a build product (git-ignored): build it once per checkout before importing the package.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
ROOT = os.path.dirname(PKG)
LIB = os.path.join(PKG, "libsinnerf_b200.so")
STAMP = os.path.join(PKG, ".libsinnerf_b200.stamp")

SOURCES = ["api.cu", "ray_kernels.cu", "field_simt.cu", "field_tc.cu", "field_bwd.cu", "wgrad_tc.cu", "dgrad_tc.cu", "optim.cu",
           "wgrad16.cu", "dgrad16.cu", "bwd16.cu", "patch_loss.cu", "warp.cu", "vit.cu"]
HEADERS = ["common.cuh", os.path.join(ROOT, "include", "sinnerf_b200.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "--shared", "-Xcompiler", "-fPIC,-O3",
    "-Xptxas", "-v",
    "--expt-relaxed-constexpr",
    "-cudart", "static",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _digest() -> str:
    h = hashlib.sha256()
    for f in SOURCES + HEADERS:
        p = f if os.path.isabs(f) else os.path.join(CSRC, f)
        for extra in ([p] if os.path.exists(p) else []):
            with open(extra, "rb") as fh:
                h.update(fh.read())
    # any other header in csrc
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cuh", ".h")) and f not in HEADERS:
            with open(os.path.join(CSRC, f), "rb") as fh:
                h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read().strip() == dig:
        return LIB
    cmd = [_nvcc()] + NVCC_FLAGS + [os.path.join(CSRC, s) for s in SOURCES] + ["-o", LIB]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    with open(os.path.join(PKG, ".build.log"), "w") as fh:
        fh.write(" ".join(cmd) + "\n" + log)
    if verbose or res.returncode != 0:
        print(log, file=sys.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed building libsinnerf_b200.so (see output above)")
    with open(STAMP, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv or "-v" in sys.argv)
    print(path)
