"""Deterministic inputs for the float64 codec and the two handlers built on it, shared by the host-compiled tests
(test_f64_on_host.py, test_f64_edges_on_host.py) and the device tests (test_gpu_f64.py), so that a disagreement on
the GPU can only come from the device build or from a path only the device has.

- `_literals`, `_patterns`, `_powers`: number texts and float64 bit patterns (seeded, no hypothesis: every run sends
  the same bytes).
- `sum_edge_payloads` / `value_edge_payloads`: hand-built json_sum / identity payloads at the edges of the device's
  domain, each with a flag that says whether the device may decline it (B9_ST_UNSUPPORTED).
- `identity_of_literal` / `json_sum_of_literal`: what the task loop answers for `{"args": [L], "kwargs": {}}` and
  `{"args": [{"values": [L]}], "kwargs": {}}`, restated without running it (test_f64_edges_on_host.py pins them
  against the oracle's task loop)."""
import json
import math
import struct
from decimal import Decimal
from fractions import Fraction

import numpy as np

COMPLETE, REJECTED = 0, 3
C_LONG_MIN, C_LONG_MAX = -(1 << 63), (1 << 63) - 1


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


# ---------------------------------------------------------------- one number, restated
def python_value_of(x: float):
    """The value json.loads makes of Go's encoding of the finite double x: Go writes an integral |x| < 1e21 as digits
    only (the shortest round-trip digits padded with zeros), which Python reads as an int; anything else reads back
    as x itself."""
    if x == int(x) and abs(x) < 1e21:
        return int(Decimal(repr(x)))
    return x


def identity_of_literal(lit: str):
    """(status, result bytes or None) of identity over `{"args": [lit], "kwargs": {}}`: Go refuses a literal that
    overflows a float64 (REJECTED); a zero value is falsy (no result)."""
    x = float(lit)
    if math.isinf(x):
        return REJECTED, None
    v = python_value_of(x)
    return COMPLETE, (json.dumps(v).encode() if v else None)


def json_sum_of_literal(lit: str):
    """(status, result bytes or None, may_decline) of json_sum over `{"args": [{"values": [lit]}], "kwargs": {}}`:
    a one-term sum is the term itself (0 + int is the int; 0 + float is the float, with -0.0 becoming 0.0, falsy
    either way). The device may decline an int outside a C long, and a literal of more than 19 significant digits."""
    st, res = identity_of_literal(lit)
    v = python_value_of(float(lit)) if st == COMPLETE else 0
    out_of_c_long = isinstance(v, int) and not C_LONG_MIN <= v <= C_LONG_MAX
    return st, res, out_of_c_long or _sig_digits(lit) > 19


def literal_may_decline(lit: str) -> bool:
    """identity: the device may decline a literal whose rounding it cannot settle (more than 19 significant digits)"""
    return _sig_digits(lit) > 19


# ---------------------------------------------------------------- edge corpora
def sdk_payload(arg_text: str, ws: str = " ") -> bytes:
    """The SDK's framing around one argument's JSON text; `ws` replaces the spaces json.dumps writes."""
    return ('{"args":' + ws + "[" + arg_text + "]," + ws + '"kwargs":' + ws + "{}}").encode("utf-8")


def _long_sum_doc(rng: np.random.Generator, n_terms: int, target_bytes: int) -> str:
    """A json_sum document of `n_terms` terms (17-digit and short floats, ints, bools) padded by an extra key to
    `target_bytes` of payload. Short terms are taken while the bytes left per term run low."""
    terms = []
    left = target_bytes - 64
    for j in range(n_terms):
        if left / (n_terms - j) < 20:
            k = int(rng.integers(0, 3))
            terms.append(("true", "false", "0.5")[k] if rng.random() < 0.3 else
                         str(int(rng.integers(-99, 1000))) if k else repr(round(float(rng.uniform(-9, 9)), 1)))
            left -= len(terms[-1]) + 2
            continue
        k = int(rng.integers(0, 6))
        if k == 0:
            terms.append(repr(float(rng.uniform(-1e3, 1e3))))
        elif k == 1:
            terms.append(repr(round(float(rng.uniform(-100, 100)), int(rng.integers(0, 4)))))
        elif k == 2:
            terms.append(str(int(rng.integers(-10 ** 9, 10 ** 9))))
        elif k == 3:
            terms.append("true" if rng.random() < 0.5 else "false")
        elif k == 4:
            terms.append("%.17g" % float(rng.uniform(-1, 1) * 10.0 ** int(rng.integers(-20, 6))))
        else:
            terms.append(repr(float(rng.uniform(1e15, 1e16))))
        left -= len(terms[-1]) + 2
    body = '"values": [' + ", ".join(terms) + "]"
    pad = target_bytes - len(sdk_payload('{"id": 7, ' + body + ', "pad": ""}'))
    assert pad >= 0, (n_terms, target_bytes)
    return '{"id": 7, ' + body + ', "pad": "' + "x" * pad + '"}'


MAX_TASK_BYTES = 1 << 20


def sum_edge_payloads():
    """[(payload, may_decline)] for json_sum."""
    out = []

    def doc(values_text: str, decline: bool = False, ws: str = " "):
        out.append((sdk_payload('{"values":' + ws + values_text + "}", ws), decline))

    # the exact int total at the edges of a C long (every term is a double Go writes back as the same digits)
    doc("[9000000000000000000, 220000000000000000, 3372036854775807]")
    doc("[-9000000000000000000, -220000000000000000, -3372036854775808]")
    doc("[9000000000000000000, 220000000000000000, 3372036854775808]", decline=True)
    doc("[-9000000000000000000, -220000000000000000, -3372036854775809]", decline=True)
    doc("[-9000000000000000000, -220000000000000000, -3372036854775808, 0.5]")
    doc("[-9000000000000000000, -220000000000000000, -3372036854775808, 1]")
    doc("[-9000000000000000000, -220000000000000000, -3372036854775808, -1]", decline=True)
    doc("[9000000000000000000, 220000000000000000, 3372036854775807, -1, 1]")
    # Go writes 2^62 as 4611686018427388000 (shortest digits, zero-padded) and -2^63 as -9223372036854776000
    doc("[-4611686018427387904, -4611686018427387904]", decline=True)
    doc("[-4611686018427387904, -4611686018427387904, 1e-300]", decline=True)
    doc("[-9223372036854775808]", decline=True)
    doc("[9223372036854775807]", decline=True)
    doc("[true, -9000000000000000000, -220000000000000000, -3372036854775808, false]")
    # an int total above 2^53 that rounds (ties to even) when the first float converts it
    for ints, fl in (([9007199254740992, 1], "0.0"), ([9007199254740992, 3], "0.5"), ([9007199254740992, 1], "-0.0"),
                     ([1152921504606846976, 64], "1.5"), ([1152921504606846976, 128], "0.5"), ([1152921504606846976, 384], "0.5"),
                     ([1152921504606846976, 128], "-0.0"), ([4611686018427387904, -512], "1e-300"),
                     ([-1152921504606846976, -384], "0.25")):
        doc("[" + ", ".join(map(str, ints)) + ", " + fl + "]")
    # int terms above 2^53 after the switch to float mode (added as a double, uncompensated)
    doc("[0.5, 9007199254740993, 18014398509481990, 100000000000000000, -3.0]")
    doc("[1e-3, 36028797018963966, 36028797018963970, -36028797018963968, 0.1]")
    doc("[0.1, 1152921504606846976, 0.2, -1152921504606846976, 0.3]")
    doc("[1.5, 9223372036854775807]", decline=True)                        # the term itself is 2^63
    doc("[1.5, 1e20]", decline=True)                                       # Go's 100000000000000000000 is beyond a C long
    doc("[1.5, 1e21, -1e21]")                                              # >= 1e21: Go writes 1e+21, a float
    # overflow to +-inf; compensation that turns into NaN is not added
    for t in ("[1e308, 1e308]", "[-1e308, -1e308]", "[1e308, 1e308, -1e308]", "[1e308, 1e308, -1e308, -1e308]",
              "[1.7976931348623157e308, 1e292]", "[-1.7976931348623157e308, -1e292]", "[1.7976931348623157e308, 9.9e291]",
              "[1e308, 1e308, 1e308, -1e308, 0.5]", "[1e308, -1e308, 1e308, 1e308]", "[0.5, 1.7976931348623157e308, 1.7976931348623157e308, 1]",
              "[1e300, 1e300, -1e300, 1e308, 1e308, -1e308, -1e308]"):
        doc(t)
    # cancellation to 0.0 and -0.0 (falsy: no result bytes)
    for t in ("[0.5, -0.5]", "[-0.0]", "[-0.0, -0.0]", "[-0.5, 0.5, -0.0]", "[0, -0.0]", "[1e16, 1.0, -1e16, -1.0]",
              "[0.1, 0.2, -0.30000000000000004]", "[-1e-320, 1e-320]", "[5e-324, -5e-324, -0.0]", "[1, -1.0]", "[true, -1.0]"):
        doc(t)
    # bools before and after the first float
    for t in ("[true, true, 0.5, false, true]", "[false, 1.5, true]", "[true]", "[true, false, true]", "[0.25, true, true, true]",
              "[true, 9007199254740992, 0.5]", "[9007199254740992, true, 0.0]"):
        doc(t)
    # the "values" key: spelled with escapes, duplicated (the last one wins), nested inside other keys
    for d in ('{"v\\u0061lues": [1.5, 2]}', '{"\\u0076alues": [0.1, 0.7]}', '{"values": [1, 2], "values": [0.25]}',
              '{"values": [0.25], "values": [1, 2]}', '{"values": [0.5], "x": {"values": [1]}}', '{"a": {"values": [9]}, "values": [0.1, 0.2]}',
              '{"x": {"values": [0.5]}}', '{"values": [1], "values": "ab"}', '{"values": "ab", "values": [0.5, 0.25]}',
              '{"values": [0.5], "v\\u0061lues": [1e300, 1e300]}', '{"Values": [0.5]}', '{"values\\u0000": [0.5]}',
              '{"values": {}}', '{"values": []}', '{"values": ""}', '{"values": [0.5, "s"]}', '{"values": [0.5, null]}',
              '{"values": [0.5, [1]]}', '{"values": [1e400]}', '{"values": [0.5], "other": -1e999}'):
        out.append((sdk_payload(d), False))
    # whitespace: none at all, and newlines / tabs / carriage returns between every token
    for ws in ("", "\n", "\t", "\r\n", " \t\n "):
        for t in ("[0.1, 0.2, 0.3]", "[1, 2, 1e16, -1e16, 0.5]", "[-9000000000000000000, -220000000000000000, -3372036854775808]"):
            sep = "," + ws
            doc("[" + ws + sep.join(t[1:-1].split(", ")) + ws + "]", ws=ws)
    # long lists: 10k-60k terms, from about 64 KiB to just under the 1 MiB largest task
    rng = np.random.default_rng(20261016)
    for n_terms, target in ((10_000, 64 << 10), (10_000, 100 << 10), (25_000, 300 << 10), (40_000, 600 << 10),
                            (60_000, MAX_TASK_BYTES - 64), (60_000, MAX_TASK_BYTES)):
        out.append((sdk_payload(_long_sum_doc(rng, n_terms, target)), False))
    assert all(len(p) <= MAX_TASK_BYTES for p, _ in out)
    return out


def _nest(depth: int, inner: str, obj_levels=()) -> str:
    """`inner` inside `depth` containers; the levels listed in obj_levels are objects {"k": ...}, the rest lists."""
    s = inner
    for d in reversed(range(depth)):
        s = '{"k%d": %s}' % (d, s) if d in obj_levels else "[" + s + "]"
    return s


def _wide(n: int, value=lambda i: str(i)) -> str:
    return "{" + ", ".join('"m%03d": %s' % (i, value(i)) for i in range(n)) + "}"


def value_edge_payloads():
    """[(payload, may_decline)] for identity."""
    out = []

    def arg(text: str, decline: bool = False, ws: str = " "):
        out.append((sdk_payload(text, ws), decline))

    # nesting: 16 levels are answered, 17 declined
    for depth in (15, 16, 17, 18):
        for objs in ((), tuple(range(0, depth, 2)), tuple(range(depth))):
            arg(_nest(depth, "1.5", objs), decline=depth > 16)
            arg(_nest(depth, '"s\\u00e9"', objs), decline=depth > 16)
    arg("[" + _nest(15, "[]") + ", 1]")                                     # an empty container needs no level
    arg("[" + _nest(16, "{}") + ", 1]", decline=True)
    # members: 64 are answered, 65 declined (also when nested)
    for n in (63, 64, 65, 100):
        arg(_wide(n), decline=n > 64)
        arg("[1, " + _wide(n, lambda i: "%d.5" % (n - i)) + "]", decline=n > 64)
        arg('{"x": ' + _wide(n, lambda i: '"v%d"' % i) + "}", decline=n > 64)
    arg("[" + ", ".join([_wide(64)] * 3) + "]")
    # duplicate keys (the last wins) and keys equal only after unescaping
    for t in ('{"a": 1, "\\u0061": 2}', '{"\\u0061": 1, "a": 2}', '{"b": 1, "a": 2, "b": 3}', '{"a": 1, "a": 2, "a": 3, "b": 0}',
              '{"/": 1, "\\/": 2}', '{"\\u00e9": 1, "é": 2.5}', '{"é": 1, "\\u00e9": 2.5}', '{"x": {"k": 1, "k": [1, {"k": 2, "k": 3}]}}',
              '{"a": 1, "b": 2, "a": 3, "c": 4, "b": 5}', '{"\\ud800": 1, "\\udfff": 2}', '{"\\ud800": 1, "\\ufffd": 2}',
              '{"\\ufffd": 1, "\\udbff": 2, "z": 0}', '{"": 1, "": 2}', '{"a\\u0000": 1, "a": 2}'):
        arg(t)
    # keys whose UTF-8 byte order differs from their UTF-16 order (Go sorts by the bytes)
    for t in ('{"\\uffff": 1, "\\ud83d\\ude00": 2}', '{"\\ud83d\\ude00": 1, "\\uffff": 2}', '{"￿": 1, "\U0001f600": 2}',
              '{"\U0001f600": 1, "￿": 2}', '{"\\ue000": 1, "\\ud800\\udc00": 2, "\\uff61": 3, "\\udbff\\udfff": 4}',
              '{"a\\uffff": 1, "a\\ud83d\\ude00": 2, "a": 3, "a\\u007f": 4, "a\\u0080": 5}', '{"é": 1, "e": 2, "z": 3, "\\u00ff": 4, "\\u0100": 5}'):
        arg(t)
    # numbers in every spelling
    nums = ["1E5", "1e5", "1e+5", "1E+5", "1e-5", "1E-5", "-1.5E-3", "-0", "-0.0", "0", "0.0", "0e10", "-0E-10", "1e-400", "-1e-400",
            "1e21", "1e22", "-1e21", "9.999999999999999e20", "999999999999999999999", "1e20", "-1e20", "123456789e15",
            "9007199254740993", "9007199254740992", "18446744073709551616", "-18446744073709551616", "2.5e+20", "1.7976931348623157e308",
            "5e-324", "2.2250738585072014E-308", "0.1", "100", "-100.000", "1.0e0", "12345678901234567890", "73786976294838206464",
            "1e-7", "1e-6", "123.456e-2", "0.000001", "1000000000000000000000.0"]
    short = [n for n in nums if _sig_digits(n) <= 19]                      # (longer ones may be declined: alone, below)
    arg("[" + ", ".join(short) + "]")
    arg(_wide(len(short), lambda i: short[i]))
    arg("[" + _wide(len(short), lambda i: "[" + short[-1 - i] + ", " + short[i] + "]") + "]")
    for n in nums:
        arg("[" + n + "]", decline=_sig_digits(n) > 19)
        arg('{"n": ' + n + "}", decline=_sig_digits(n) > 19)
    arg("[1e400]")                                                         # overflow: Go refuses the payload
    arg('{"a": [1, {"b": -1e309}]}')
    # lone surrogates inside nested strings (Go reads each as U+FFFD)
    for t in ('["\\ud800", {"k": "\\udc00x"}, [["a\\udbff"]]]', '{"k": ["\\udfff\\ud800", "\\ud83d\\ude00", "\\ud83d"]}',
              '[["\\ud800\\ud800"], "x\\udc00\\udc00y", {"\\udc00": "\\ud800"}]'):
        arg(t)
    # whitespace variants inside the value
    for ws in ("", "\n", "\t", "\r\n  "):
        arg("{" + ws + '"b"' + ws + ":" + ws + "[" + ws + "1.5" + ws + "," + ws + "true" + ws + "]" + ws + "," + ws + '"a"' + ws + ":" + ws
            + "{" + ws + "}" + ws + "}", ws=ws)
        arg("[" + ws + "[" + ws + "]" + ws + "," + ws + '"x"' + ws + "," + ws + "-0" + ws + "," + ws + "null" + ws + "]", ws=ws)
    # containers of 2 KiB to 512 KiB: larger than every stage buffer
    rng = np.random.default_rng(20261017)
    leaves = ["1.5", "-0.0", "1e21", "123456789012345678", '"caf\\u00e9"', '"\\ud83d\\ude00"', "true", "null", "[]", "{}", '"x<y"',
              "0.30000000000000004", "-7", "1E-7"]
    for target in (2 << 10, 8 << 10, 40 << 10, 64 << 10, 200 << 10, 512 << 10):
        items, size = [], 2
        while size < target:
            k = int(rng.integers(0, 4))
            if k == 0:
                it = leaves[int(rng.integers(0, len(leaves)))]
            elif k == 1:
                it = repr(float(rng.uniform(-1e6, 1e6)))
            elif k == 2:
                it = _wide(int(rng.integers(1, 9)), lambda i: leaves[int(rng.integers(0, len(leaves)))])
            else:
                it = "[" + ", ".join(repr(float(x)) for x in rng.standard_normal(int(rng.integers(1, 12)))) + "]"
            items.append(it)
            size += len(it) + 2
        arg("[" + ", ".join(items) + "]")
        per = (target - 64) // 64                                          # an object of 64 long members
        arg(_wide(64, lambda i: "[" + ", ".join(["%d.25" % i] * max(1, per // 6)) + "]"))
    return out
