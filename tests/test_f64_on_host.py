"""The device's float64 codec (beta9_b200/csrc/f64_device.cuh), compiled for the host by tests/host_shim/f64_shim.cpp,
against Python: the parser against float() (and its overflow decisions against number_overflows_f64), the shortest
digits and the three writers against repr(), json.dumps and the oracle's restatement of Go's float encoder.

B9_F64_PATTERNS (default 10M) sets how many random bit patterns the repr() comparison covers; the Go-encoder and
Go->Python comparisons, whose expected texts come from slower Python code, cover a fifth of that."""
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np
import pytest

from oracle.pyoracle.gojson import go_format_float64
from tests.f64_corpus import _bits, _literals, _patterns, _powers, _sig_digits

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_shim", "f64_shim.cpp")
SO = os.path.join(HERE, "host_shim", "libf64shim.so")
GXX = os.environ.get("CXX", "g++")
N_PATTERNS = int(os.environ.get("B9_F64_PATTERNS", 10_000_000))


@pytest.fixture(scope="module")
def f64():
    csrc = os.path.join(os.path.dirname(HERE), "beta9_b200", "csrc")
    deps = [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".h"))]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max([os.path.getmtime(SRC)] + [os.path.getmtime(d) for d in deps]):
        r = subprocess.run([GXX, "-O2", "-std=c++17", "-shared", "-fPIC", "-o", SO, SRC], capture_output=True, text=True)
        if r.returncode:
            pytest.skip("no host C++ compiler for the shim: " + r.stderr[-300:])
    lib = C.CDLL(SO)
    u64p, u8p = np.ctypeslib.ndpointer(np.uint64, flags="C"), np.ctypeslib.ndpointer(np.uint8, flags="C")
    lib.b9_f64_parse_batch.argtypes = [C.c_char_p, u64p, C.c_uint64, u64p, u8p, u8p]
    lib.b9_f64_format_batch.argtypes = [u64p, C.c_uint64, C.c_int, C.c_char_p]
    lib.b9_f64_format_batch.restype = C.c_uint64

    class F64:
        @staticmethod
        def parse(lits):
            enc = [s.encode() for s in lits]
            off = np.zeros(len(enc) + 1, np.uint64)
            np.cumsum([len(b) for b in enc], out=off[1:])
            bits = np.zeros(len(enc), np.uint64)
            ok = np.zeros(len(enc), np.uint8)
            over = np.zeros(len(enc), np.uint8)
            lib.b9_f64_parse_batch(b"".join(enc), off, len(enc), bits, ok, over)
            return bits, ok, over

        @staticmethod
        def format(bits: np.ndarray, which: int):
            bits = np.ascontiguousarray(bits, dtype=np.uint64)
            buf = C.create_string_buffer(32 * len(bits) + 64)
            n = lib.b9_f64_format_batch(bits, len(bits), which, buf)
            assert n or not len(bits), "sizing and writing passes disagree"
            return buf.raw[:n].decode().split("\n")[:-1]
    return F64


def test_parser_against_float(f64):
    lits = _literals()
    assert len(lits) >= 1_000_000
    bits, ok, over = f64.parse(lits)
    declined_long = 0
    for lit, b, k, ov in zip(lits, bits.tolist(), ok.tolist(), over.tolist()):
        want = float(lit)
        assert bool(ov) == math.isinf(want), (lit, ov)           # number_overflows_f64 == strconv's ErrRange
        if not k:
            assert _sig_digits(lit) > 19, lit                     # never declined with <= 19 significant digits
            declined_long += 1
            continue
        assert b == _bits(want), (lit, hex(b), want)
    n_long = sum(1 for s in lits if _sig_digits(s) > 19)
    print(f"\nf64_parse: {len(lits)} literals, {n_long} with > 19 significant digits, {declined_long} of those declined")


def _py_float_json(x: float) -> str:
    return json.dumps(x)


def test_shortest_digits_and_python_repr(f64):
    """py_json_float == json.dumps(float) == repr for finite values: pins f64_shortest's digits."""
    chunk = 1_000_000
    done = 0
    for seed in range(0, max(1, N_PATTERNS // chunk)):
        b = _patterns(chunk, 1000 + seed)
        got = f64.format(b, 1)
        want = list(map(repr, b.view(np.float64).tolist()))
        if got != want:
            bad = next(i for i in range(len(want)) if got[i] != want[i])
            raise AssertionError((hex(int(b[bad])), got[bad], want[bad]))
        done += len(b)
    p = _powers()
    assert f64.format(p, 1) == list(map(_py_float_json, p.view(np.float64).tolist()))
    nonfinite = np.array([_bits(math.inf), _bits(-math.inf), _bits(math.nan), 0xFFF8000000000001], np.uint64)
    assert f64.format(nonfinite, 1) == ["Infinity", "-Infinity", "NaN", "NaN"]
    assert done >= min(N_PATTERNS, 10_000_000) * 0.99


def _go_then_python(x: float) -> str:
    return json.dumps(json.loads(go_format_float64(x)))


def test_go_float_encoder_and_python_reading(f64):
    n = max(1, N_PATTERNS // 5)
    for seed in range(0, max(1, n // 1_000_000)):
        b = _patterns(min(n, 1_000_000), 2000 + seed)
        xs = b.view(np.float64).tolist()
        assert f64.format(b, 0) == list(map(go_format_float64, xs))
        if seed == 0:
            assert f64.format(b[:300_000], 2) == list(map(_go_then_python, xs[:300_000]))
    p = _powers()
    xs = p.view(np.float64).tolist()
    assert f64.format(p, 0) == list(map(go_format_float64, xs))
    assert f64.format(p, 2) == list(map(_go_then_python, xs))
    # the texts of the identity table of the feature's description
    table = {1.5: "1.5", 123.0: "123", 1e20: "100000000000000000000", 1e21: "1e+21", 1e-7: "1e-07",
             73786976294838206464.0: "73786976294838210000", -0.0: "0", 1e16: "10000000000000000", 0.1: "0.1"}
    for x, want in table.items():
        assert f64.format(np.array([_bits(x)], np.uint64), 2) == [want], x
