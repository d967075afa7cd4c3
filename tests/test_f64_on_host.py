"""The device's float64 codec (beta9_b200/csrc/f64_device.cuh), compiled for the host by tests/host_shim/f64_shim.cpp,
against Python: the parser against float() (and its overflow decisions against number_overflows_f64), the shortest
digits and the three writers against repr(), json.dumps and the oracle's restatement of Go's float encoder.

B9_F64_PATTERNS (default 10M) sets how many random bit patterns the repr() comparison covers; the Go-encoder and
Go->Python comparisons, whose expected texts come from slower Python code, cover a fifth of that."""
import ctypes as C
import json
import math
import os
import struct
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from oracle.pyoracle.gojson import go_format_float64

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


def _bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def _sig_digits(lit: str) -> int:
    m = lit.lstrip("-").split("e")[0].split("E")[0].replace(".", "").lstrip("0")
    return len(m)


def _literals():
    rng = np.random.default_rng(20261015)
    pats = rng.integers(0, 1 << 64, size=280_000, dtype=np.uint64)
    xs = [x for x in pats.view(np.float64).tolist() if math.isfinite(x)]
    out = []
    for x in xs:
        out += [repr(x), "%.17g" % x, "%.25e" % x]
    specials = [5e-324, 1e-323, 2.2250738585072009e-308, 2.2250738585072014e-308, 1.7976931348623157e308, 2.0 ** 53 - 1, 2.0 ** 53,
                2.0 ** 53 + 2, 1e22, 1e23, 0.1, 0.3, 1.5, 123.0, 1e20, 1e21, 1e-7]
    for x in specials:
        out += [repr(x), "%.17g" % x, "%.25e" % x, "%.40e" % x]
    out += ["9007199254740993", "9007199254740991", "9007199254740992", "1e22", "1e23", "8.98846567431158e307", "0", "-0", "0.0", "-0.0",
            "1e400", "-1e400", "1e-400", "-1e-400", "1e-350", "1e-342", "1e-343", "1e308", "1e309", "1.7976931348623158e308",
            "1.7976931348623159e308", "179769313486231580793728971405303415079934132710037826936173778980444968292764750946649017977587207096330286416692887910946555547851940402630657488671505820681908902000708383676273854845817711531764475730270069855571366959622842914819860834936475292719074168444365510704342711559699508093042880177904174497791",
            "2.4703282292062327e-324", "2.4703282292062328e-324", "4.9406564584124654e-324", "1e-5", "0.000001", "0." + "0" * 300 + "1",
            "1" + "0" * 300, "00", "1.00000000000000000000000000000000000000000"]
    out = [s for s in out if not s.startswith("00")]
    for _ in range(60_000):                                 # 1..19 digits, exponents -400..400
        nd = int(rng.integers(1, 20))
        w = "".join(map(str, rng.integers(0, 10, size=nd).tolist())).lstrip("0") or "1"
        out.append("%se%d" % (w, int(rng.integers(-400, 401))))
    # subnormals
    sub = rng.integers(1, 1 << 52, size=20_000, dtype=np.uint64).view(np.float64).tolist()
    out += [repr(x) for x in sub] + ["%.17g" % x for x in sub]
    # 20-40 digit literals at exact midpoints between adjacent doubles, and one unit of the last digit either side
    for _ in range(40_000):
        m = int(rng.integers(1 << 52, 1 << 53))
        if rng.random() < 0.5:
            e = int(rng.integers(11, 72))                   # integers: (2m+1) 2^(e-1)
            mid = Fraction((2 * m + 1) << (e - 1))
        else:
            j = int(rng.integers(1, 23))                    # fractions with j+1 decimals: (2m+1) 2^-(j+1)
            mid = Fraction(2 * m + 1, 1 << (j + 1))
        den_pow = 0
        while (mid * 10 ** den_pow).denominator != 1:
            den_pow += 1
        digits = str((mid * 10 ** den_pow).numerator)
        for delta in (0, -1, 1):
            d = str(int(digits) + delta)
            lit = d + "e-%d" % den_pow if den_pow else d
            if 20 <= _sig_digits(lit) <= 40:
                out.append(("-" if rng.random() < 0.3 else "") + lit)
    return out


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


def _patterns(n: int, seed: int):
    rng = np.random.default_rng(seed)
    b = rng.integers(0, 1 << 64, size=n, dtype=np.uint64)
    return b[(b & np.uint64(0x7FF0000000000000)) != np.uint64(0x7FF0000000000000)]


def _powers():
    xs = [2.0 ** e for e in range(-1074, 1024)] + [float("1e%d" % e) for e in range(-323, 309)]
    xs += [5e-324 * k for k in range(1, 50)] + [1.7976931348623157e308, 2.2250738585072014e-308, 1e21, 1e-6, 1e16, 1e-4, 1e-5]
    xs += [math.nextafter(x, math.inf) for x in list(xs)] + [math.nextafter(x, 0.0) for x in list(xs)]
    xs = [x for x in xs if math.isfinite(x)]
    xs += [-x for x in xs] + [0.0, -0.0]
    return np.array([_bits(x) for x in xs], dtype=np.uint64)


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
