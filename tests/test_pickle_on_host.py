"""The function path's pickle codec on a CPU (B9_DRAIN_PICKLE_FULL): pickle_device.cuh compiled for the host by
tests/host_shim/pickle_shim.cpp, against the oracle's runner loop (funcloop.run_function_task: cloudpickle.loads ->
handler -> cloudpickle.dumps) for every handler, byte for byte and status for status. Every UNSUPPORTED of the structured
corpus has a documented reason (tests/pickle_corpus.declined); random byte mutations are held to "never a wrong answer"."""
import base64
import ctypes as C
import json
import os
import subprocess

import cloudpickle
import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from oracle.pyoracle import funcloop
from tests import pickle_corpus as PC

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_shim", "pickle_shim.cpp")
SO = os.path.join(HERE, "host_shim", "libpickleshim.so")
GXX = os.environ.get("CXX", "g++")
OK, ERROR, UNSUPPORTED = 0, 1, 4
H_ID = {"identity": 0, "crc32": 1, "vadd_f32": 2, "json_sum": 3}


@pytest.fixture(scope="module")
def pk():
    csrc = os.path.join(os.path.dirname(HERE), "beta9_b200", "csrc")
    deps = [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".h"))]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max([os.path.getmtime(SRC)] + [os.path.getmtime(d) for d in deps]):
        r = subprocess.run([GXX, "-O2", "-std=c++17", "-shared", "-fPIC", "-o", SO, SRC], capture_output=True, text=True)
        if r.returncode:
            pytest.skip("no host C++ compiler for the shim: " + r.stderr[-300:])
    lib = C.CDLL(SO)
    u64p, u8p = np.ctypeslib.ndpointer(np.uint64, flags="C"), np.ctypeslib.ndpointer(np.uint8, flags="C")
    lib.b9_pk_batch.argtypes = [C.c_char_p, u64p, C.c_uint32, C.c_int, u8p, C.c_void_p, u64p]
    lib.b9_pk_batch.restype = C.c_uint64

    def batch(blobs, handler):
        """[(status, result bytes or None)] per blob"""
        n = len(blobs)
        off = np.zeros(n + 1, np.uint64)
        np.cumsum([len(b) for b in blobs], out=off[1:])
        blob = b"".join(blobs)
        status, out_off = np.zeros(max(n, 1), np.uint8), np.zeros(n + 1, np.uint64)
        total = lib.b9_pk_batch(blob, off, n, H_ID[handler], status, None, out_off)
        out = np.zeros(total + 1, np.uint8)
        lib.b9_pk_batch(blob, off, n, H_ID[handler], status, out.ctypes.data, out_off)
        raw = out.tobytes()
        return [(int(status[i]), raw[int(out_off[i]):int(out_off[i + 1])] if status[i] == OK else None) for i in range(n)]
    return batch


def oracle(blob, handler):
    st_, res = funcloop.run_function_task(blob, handler)
    return (OK, res) if st_ == funcloop.COMPLETE else (ERROR, None)


def check(pk, blobs, handler, strict=True):
    """strict: every UNSUPPORTED has a documented reason. Returns the number of answered blobs."""
    answered = 0
    for b, got in zip(blobs, pk(blobs, handler)):
        if got[0] == UNSUPPORTED:
            if strict:
                assert PC.declined(b, handler), (handler, b[:120])
            continue
        answered += 1
        assert got == oracle(b, handler), (handler, b[:120])
    return answered


@pytest.mark.parametrize("handler", PC.HANDLERS)
def test_structured_corpus(pk, handler):
    blobs = PC.structured_blobs()
    assert check(pk, blobs, handler) > len(blobs) // 2


def golden_cases():
    return json.load(open(os.path.join(HERE, "golden", "ref_function_full_golden.json")))["cases"]


def golden_want(c, handler):
    want = c["results"][handler]
    return (OK, base64.b64decode(want["result_pickle"])) if want["ok"] else (ERROR, None)


@pytest.mark.parametrize("handler", PC.HANDLERS)
def test_reference_full_golden(pk, handler):
    """what the reference's own function runner returned (make_ref_function_full_golden.py): the oracle restates it, the
    codec answers it or declines with a documented reason; the domain's inputs are answered"""
    cases = golden_cases()
    blobs = [base64.b64decode(c["args_pickle"]) for c in cases]
    answered = 0
    for c, b, got in zip(cases, blobs, pk(blobs, handler)):
        want = golden_want(c, handler)
        assert oracle(b, handler) == want, c["input_repr"]
        if got[0] == UNSUPPORTED:
            assert PC.declined(b, handler), c["input_repr"]
            continue
        answered += 1
        assert got == want, (handler, c["input_repr"])
    assert answered >= len(cases) - 3, handler


def test_domain_is_answered(pk):
    """what the issue's domain promises is answered, not declined"""
    docs = PC.sdk_blobs(100)
    for h in ("identity", "json_sum"):
        assert all(s != UNSUPPORTED for s, _ in pk(docs[:100], h)), h
    cases = [PC.frame_one(v) for v in [0, 255, 256, 65535, 65536, 2**31, -2**31 - 1, 2**63, 10**30, -0.0, float("nan"),
                                        list(range(2000)), [str(i) for i in range(300)], {str(i): i for i in range(64)}]]
    assert all(s == OK for s, _ in pk(cases, "identity"))
    assert pk([PC.frame_one({str(i): i for i in range(65)})], "identity")[0][0] == UNSUPPORTED
    assert pk([PC.frame_one(0)], "identity")[0][1] == bytes.fromhex("80054b002e")


def test_singletons_and_sharing(pk):
    for b in PC.hand_built()[:8]:
        got = pk([b], "identity")[0]
        assert got == oracle(b, "identity"), b


def test_truncations(pk):
    blobs = [b for b in PC.structured_blobs() if len(b) < 2000][:150]
    cut = [b[:k] for b in blobs for k in range(0, len(b), max(1, len(b) // 20))]
    for h in PC.HANDLERS:
        check(pk, cut, h, strict=False)


@pytest.mark.parametrize("handler", PC.HANDLERS)
def test_random_mutations(pk, handler):
    blobs = PC.mutations(PC.structured_blobs(), 30_000 // 4, seed=11 + H_ID[handler])
    check(pk, blobs, handler, strict=False)


_scalars = st.one_of(st.none(), st.booleans(), st.integers(), st.floats(allow_nan=True), st.text(max_size=20),
                     st.binary(max_size=20))
_keys = st.one_of(st.text(max_size=8), st.integers(-5, 300), st.binary(max_size=4), st.none(), st.booleans())
_values = st.recursive(_scalars, lambda ch: st.one_of(st.lists(ch, max_size=6), st.tuples(ch, ch),
                                                      st.dictionaries(_keys, ch, max_size=6)), max_leaves=40)


@settings(max_examples=400, deadline=None, suppress_health_check=[HealthCheck.too_slow])
@given(v=_values)
def test_hypothesis_values(pk, v):
    b = funcloop.frame_call(v)
    for h in PC.HANDLERS:
        got = pk([b], h)[0]
        if got[0] == UNSUPPORTED:
            assert PC.declined(b, h), (h, v)
        else:
            assert got == oracle(b, h), (h, v)
    doc = funcloop.frame_call({"values": v if isinstance(v, (list, tuple)) else [v]})
    got = pk([doc], "json_sum")[0]
    if got[0] != UNSUPPORTED:
        assert got == oracle(doc, "json_sum"), v


def test_identity_results_unpickle(pk):
    vals = PC.plain_values()[:60]
    for v, (s, res) in zip(vals, pk([PC.frame_one(v) for v in vals], "identity")):
        if s == OK:
            assert res == cloudpickle.dumps(v), repr(v)[:80]
