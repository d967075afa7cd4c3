"""The loopback NCCL stand-in (tests/loopback_nccl/loopback_nccl.cpp) builds with g++ alone and exports every NCCL
symbol libb9gpu.so loads, so that tests/test_gpu_rebalance_loopback.py can stand it in for NCCL on one GPU."""
import ctypes as C
import os
import re
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "loopback_nccl", "loopback_nccl.cpp")
LIB_SRC = os.path.join(os.path.dirname(HERE), "beta9_b200", "csrc", "b9gpu.cu")


def nccl_symbols_the_library_loads():
    with open(LIB_SRC) as f:
        return sorted(set(re.findall(r'SYM\(\s*\w+\s*,\s*"(nccl\w+)"\s*\)', f.read())))


def test_loopback_builds_and_exports_the_nccl_symbols(tmp_path):
    so = os.path.join(str(tmp_path), "libloopback_nccl.so")
    r = subprocess.run([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-Wall", "-Werror", "-shared", "-fPIC", "-o", so, SRC, "-ldl", "-lpthread"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    names = nccl_symbols_the_library_loads()
    assert names == sorted(["ncclGetUniqueId", "ncclCommInitRank", "ncclCommDestroy", "ncclAllGather", "ncclSend", "ncclRecv",
                            "ncclGroupStart", "ncclGroupEnd", "ncclGetErrorString"])
    lib = C.CDLL(so)                       # loads without a GPU: libcuda.so.1 is opened on the first collective only
    for name in names + ["lb_log_count", "lb_log_get"]:
        getattr(lib, name)                 # AttributeError if it is not exported
    lib.lb_log_count.restype = C.c_long
    assert lib.lb_log_count(0) == 0
    lib.ncclGetErrorString.restype = C.c_char_p
    assert lib.ncclGetErrorString(0)
