"""Builds libb9gpu.so (the C-ABI library, include/b9gpu.h) in-tree with nvcc for sm_90a (H100).

    python -m beta9_b200.build [--force] [--ptxas-v]

nvcc cross-compiles without a GPU. The .so is a build product (git-ignored).
"""
from __future__ import annotations

import os
import subprocess
import sys
from typing import List

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
SO = os.path.join(PKG, "libb9gpu.so")
SOURCES = ["b9gpu.cu", "wire_full.cu", "function_drain.cu", "endpoint_drain.cu", "callback_sign.cu", "callback_runners.cu"]   # (all but b9gpu.cu: kernels in modules of their own)
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

FLAGS = [
    "-O3", "-std=c++17", "-lineinfo",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-Xcompiler", "-fPIC,-O3,-Wall,-Wno-unused-function",
    "--shared", "-cudart", "static",
]


def _deps() -> List[str]:
    out = [os.path.join(ROOT, "include", "b9gpu.h")]
    for f in os.listdir(CSRC):
        if f.endswith((".cu", ".cuh", ".h", ".hpp", ".cpp")):
            out.append(os.path.join(CSRC, f))
    return out


def needs_build() -> bool:
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    return any(os.path.getmtime(d) > t for d in _deps())


def build(force: bool = False, verbose_ptxas: bool = False) -> str:
    if not force and not needs_build():
        return SO
    if not os.path.exists(NVCC):
        raise RuntimeError(f"nvcc not found at {NVCC}: libb9gpu.so cannot be built (there is no CPU fallback)")
    cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose_ptxas else []) + \
          ["-o", SO] + [os.path.join(CSRC, s) for s in SOURCES] + ["-ldl", "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose_ptxas or r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    return SO


def build_variant(name: str, defines: List[str]) -> str:
    """An alternative build for A/B timing on one box: ab_builds/<name>.so compiled with extra -D switches
    (selected at run time with B9GPU_LIB=...). ab_builds/ is git-ignored."""
    out_dir = os.path.join(ROOT, "ab_builds")
    os.makedirs(out_dir, exist_ok=True)
    out = os.path.join(out_dir, name + ".so")
    cmd = [NVCC] + FLAGS + ["-D" + d for d in defines] + ["-o", out] + [os.path.join(CSRC, s) for s in SOURCES] + ["-ldl", "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    return out


if __name__ == "__main__":
    if "--variant" in sys.argv:          # python -m beta9_b200.build --variant NAME [-DX=1 ...]
        i = sys.argv.index("--variant")
        print(build_variant(sys.argv[i + 1], [a[2:] for a in sys.argv[i + 2:] if a.startswith("-D")]))
        sys.exit(0)
    print(build(force="--force" in sys.argv, verbose_ptxas="--ptxas-v" in sys.argv))
