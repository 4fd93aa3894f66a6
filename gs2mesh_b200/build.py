"""Builds gs2mesh_b200/libgs2mesh_b200.so (sm_90a only: H100) in-tree with nvcc.

nvcc cross-compiles without a GPU, so the library can be built on a machine without one.
"""
from __future__ import annotations

import os
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG_DIR)
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "libgs2mesh_b200.so")
SOURCES = ["gsb_raster.cu", "gsb_tsdf.cu", "gsb_mesh.cu", "gsb_reduce.cu", "gsb_eval.cu", "gsb_cull.cu"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-ldl"]


def _sources():
    return [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def _deps():
    deps = _sources() + [os.path.join(ROOT, "include", "gs2mesh_b200.h")]
    deps += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".h") or f.endswith(".cuh")]
    return deps


def needs_build() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    built = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(d) > built for d in _deps())


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB_PATH] + _sources()
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        sys.stderr.write(proc.stdout + proc.stderr)
        raise RuntimeError("nvcc failed building libgs2mesh_b200.so")
    if verbose:
        sys.stderr.write(proc.stderr)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
