"""Builds libb9gpu.so (the C-ABI library, include/b9gpu.h) in-tree with nvcc for sm_90a (H100).

    python -m beta9_b200.build [--force] [--ptxas-v]

nvcc cross-compiles without a GPU. The .so is a build product (git-ignored).
"""
from __future__ import annotations

import os
import subprocess
import sys
from typing import List, Optional

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
SO = os.path.join(PKG, "libb9gpu.so")
SOURCES = ["b9gpu.cu", "wire_full.cu", "endpoint_drain.cu", "drain_passes.cu"]   # (all but b9gpu.cu: kernels in modules of their own)
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


HANDLER_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-cubin", "-gencode", "arch=compute_90a,code=sm_90a"]
EXAMPLE_HANDLERS = os.path.join(ROOT, "examples", "handlers", "handlers.cu")
EXAMPLE_CUBIN = os.path.join(PKG, "example_handlers.cubin")     # build product (git-ignored), loaded with b9_handler_load


def handler_abi_version() -> int:
    """B9_HANDLER_ABI_VERSION (drain_kernel.cuh): the version the entry names of a handler image carry."""
    import re
    with open(os.path.join(CSRC, "drain_kernel.cuh")) as f:
        return int(re.search(r"#define B9_HANDLER_ABI_VERSION (\d+)", f.read()).group(1))


def compile_handlers(src: str, out: str, includes: Optional[List[str]] = None, force: bool = False) -> str:
    """Compiles a translation unit of B9_HANDLER lines (include/b9gpu_handler.cuh) to an sm_90a cubin for
    b9_handler_load, with the library's flags and include path. As build(): nothing is done while `out` is newer than
    `src`, the headers next to it and the library's device headers."""
    src, out = os.path.abspath(src), os.path.abspath(out)
    here = os.path.dirname(src)
    deps = [src] + _deps() + [os.path.join(ROOT, "include", "b9gpu_handler.cuh")] + \
        [os.path.join(here, f) for f in os.listdir(here) if f.endswith((".cuh", ".h"))]
    if not force and os.path.exists(out) and not any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        return out
    if not os.path.exists(NVCC):
        raise RuntimeError(f"nvcc not found at {NVCC}: {src} cannot be compiled")
    inc = ["-I" + os.path.join(ROOT, "include"), "-I" + here] + ["-I" + d for d in (includes or [])]
    tmp = out + ".tmp"
    r = subprocess.run([NVCC] + HANDLER_FLAGS + inc + ["-o", tmp, src], capture_output=True, text=True)
    if r.returncode:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    os.replace(tmp, out)
    return out


def build_examples(force: bool = False) -> str:
    """The example handlers (examples/handlers) as beta9_b200/example_handlers.cubin, so that runs need no nvcc."""
    return compile_handlers(EXAMPLE_HANDLERS, EXAMPLE_CUBIN, force=force)


TEST_HANDLERS = os.path.join(ROOT, "tests", "handlers", "contract.cu")
TEST_CUBIN = os.path.join(ROOT, "tests", "handlers", "contract.cubin")   # build product (git-ignored)
CONTAINER_HANDLERS = os.path.join(ROOT, "tests", "handlers", "containers.cu")
CONTAINER_CUBIN = os.path.join(ROOT, "tests", "handlers", "containers.cubin")   # build product (git-ignored)


def build_test_handlers(force: bool = False) -> str:
    """The test-only handlers (tests/handlers) as tests/handlers/contract.cubin and containers.cubin, so that the GPU
    tests need no nvcc. Returns the first."""
    compile_handlers(CONTAINER_HANDLERS, CONTAINER_CUBIN, force=force)
    return compile_handlers(TEST_HANDLERS, TEST_CUBIN, force=force)


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
    print(build_examples(force="--force" in sys.argv))
    print(build_test_handlers(force="--force" in sys.argv))
