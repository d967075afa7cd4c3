"""CPU checks of b9_cancel's shared key order (beta9_b200/csrc/cancel.cuh): the key helper, the host sort and
de-duplication, and the fence search cancel_kernel runs, compiled with g++ and compared with Python's byte order and set
membership. A host sort by bytes with a device compare of differently ordered words would find nothing and raise no
error; these tests are what catches that."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_shim", "cancel_shim.cpp")
SO = os.path.join(HERE, "host_shim", "libcancel.so")
HDR = os.path.join(os.path.dirname(HERE), "beta9_b200", "csrc", "cancel.cuh")
GXX = os.environ.get("CXX", "g++")
FENCE = 2048                                      # CANCEL_FENCE_MAX


@pytest.fixture(scope="module")
def cx():
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(SRC), os.path.getmtime(HDR)):
        r = subprocess.run([GXX, "-O2", "-std=c++17", "-shared", "-fPIC", "-o", SO, SRC], capture_output=True, text=True)
        if r.returncode:
            pytest.skip("no host C++ compiler for the shim: " + r.stderr[-300:])
    lib = C.CDLL(SO)
    lib.b9_cx_key.argtypes = [C.c_void_p, C.c_void_p]
    lib.b9_cx_key.restype = None
    lib.b9_cx_sort_unique.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    lib.b9_cx_sort_unique.restype = C.c_uint32
    lib.b9_cx_find.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
    lib.b9_cx_find.restype = C.c_uint32
    return lib


def as_ids(lst):
    return np.frombuffer(b"".join(lst), np.uint8).reshape(-1, 16) if lst else np.zeros((0, 16), np.uint8)


def sort_unique(cx, ids):
    n = ids.shape[0]
    keys = np.zeros((max(n, 1), 2), np.uint64)
    which = np.zeros(max(n, 1), np.uint32)
    k = cx.b9_cx_sort_unique(ids.ctypes.data, n, keys.ctypes.data, which.ctypes.data)
    return keys[:k], which[:n]


def key_bytes(keys):
    """(hi, lo) keys back to the 16 bytes they stand for (big-endian)."""
    return [int(h).to_bytes(8, "big") + int(lo).to_bytes(8, "big") for h, lo in keys]


def edge_ids():
    out = [bytes(16), b"\xff" * 16]
    base = bytes(range(16))
    for pos in (0, 3, 4, 7, 8, 11, 12, 15):       # byte 0, byte 15, both sides of the 4- and 8-byte boundaries
        for v in (0x00, 0x01, 0x7F, 0x80, 0xFE, 0xFF):
            b = bytearray(base); b[pos] = v; out.append(bytes(b))
            z = bytearray(16); z[pos] = v; out.append(bytes(z))
            f = bytearray(b"\xff" * 16); f[pos] = v; out.append(bytes(f))
    return list(dict.fromkeys(out))


def test_key_is_big_endian_memcmp_order(cx):
    rng = np.random.default_rng(1)
    ids = [rng.bytes(16) for _ in range(500)] + edge_ids()
    out = np.zeros(2, np.uint64)
    for b in ids:
        cx.b9_cx_key(b, out.ctypes.data)
        assert int(out[0]) == int.from_bytes(b[:8], "big") and int(out[1]) == int.from_bytes(b[8:], "big"), b.hex()


@pytest.mark.parametrize("case", ["random", "edges", "duplicates"])
def test_sort_unique_equals_sorted_set(cx, case):
    rng = np.random.default_rng(2)
    if case == "random":
        lst = [rng.bytes(16) for _ in range(20_000)]
    elif case == "edges":
        lst = edge_ids()
    else:
        pool = [rng.bytes(16) for _ in range(300)] + edge_ids()
        lst = [pool[int(i)] for i in rng.integers(0, len(pool), 5000)]
    keys, which = sort_unique(cx, as_ids(lst))
    want = sorted(set(lst))
    assert key_bytes(keys) == want
    for i, b in enumerate(lst):                    # every caller's id maps to its own key
        assert want[int(which[i])] == b


@pytest.mark.parametrize("n", [1, 2, FENCE - 1, FENCE, FENCE + 1, 100_000])
def test_fence_search_equals_membership(cx, n):
    rng = np.random.default_rng(n)
    edges = edge_ids()
    pool = [rng.bytes(16) for _ in range(n)]
    if n >= len(edges):
        pool[:len(edges)] = edges
    req = pool[:n]
    absent = [rng.bytes(16) for _ in range(2000)]
    # near misses: a requested id with its first or last byte, or a byte at a word boundary, off by one
    for b in req[:500]:
        for pos in (0, 3, 4, 7, 8, 15):
            m = bytearray(b); m[pos] = (m[pos] + 1) & 0xFF; absent.append(bytes(m))
    queries = req + absent + [bytes(16), b"\xff" * 16]
    at = np.zeros(len(queries), np.int64)
    req_a, q_a = as_ids(req), as_ids(queries)
    stride = cx.b9_cx_find(req_a.ctypes.data, n, q_a.ctypes.data, len(queries), at.ctypes.data)
    assert len(set(req)) == n
    assert (n + stride - 1) // stride <= FENCE and (stride == 1 or (n + stride // 2 - 1) // (stride // 2) > FENCE)
    want = sorted(set(req))
    index = {b: i for i, b in enumerate(want)}
    for q, a in zip(queries, at):
        assert int(a) == index.get(q, -1), (q.hex(), int(a))
