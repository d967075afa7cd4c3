"""identity over numbers and non-empty lists / objects, and json_sum over float data: the device's sequential path
(tests/host_shim/host_parse.cpp) against the oracle's task loop, on a CPU."""
import json
import math
import sys

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from oracle.pyoracle import loop
from tests.test_device_parser_on_host import parser  # noqa: F401  (the host-compiled parser + handlers)

HANDLERS = {"identity": 0, "json_sum": 3}
CODE = {"COMPLETE": 0, "ERROR": 1, "RETRY": 2, "REJECTED": 3}

TABLE_IDENTITY = [
    (b"1.5", b"1.5"), (b"123.0", b"123"), (b"1e20", b"100000000000000000000"), (b"1e21", b"1e+21"), (b"1e-7", b"1e-07"),
    (b"73786976294838206464", b"73786976294838210000"), (b"-0.0", None), (b"1e-400", None),
    (b'{"b": 1, "a": 2.50, "b": [0.1, -0.0]}', b'{"a": 2.5, "b": [0.1, 0]}'),
    ('["é", "<", 1e16]'.encode(), b'["\\u00e9", "<", 10000000000000000]'),
]
TABLE_SUM = [
    (b"[0.1, 0.2, 0.3]", b"0.6"), (b"[1, 0.1, 2, 1e16, -1e16]", b"4.0"), (b"[1e308, 1e308]", b"Infinity"), (b"[0.5, -0.5]", None),
    (b"[1e300, -1e300, 0.25]", b"0.25"), (b"[true, 0.5, false]", b"1.5"), (b"[1e308, 1e308, -1e308, -1e308]", b"Infinity"),
]
# Go writes 1e20 as digits, so Python sums the int 100000000000000000000 (beyond a C long) and then 0.5 -> 1e+20: the device
# declines sums that leave the C long range
TABLE_SUM_DECLINED = [b"[1e20, 0.5]"]


def _payload_tok(tok: bytes) -> bytes:
    return b'{"args": [' + tok + b'], "kwargs": {}}'


def _check(parser, payloads, handler, allow_decline=0.0):
    ids = [bytes([i & 255]) * 16 for i in range(len(payloads))]
    want = loop.run_task_loop(payloads, ids, handler)
    declined = 0
    for b, w in zip(payloads, want):
        st_, res = parser.run(b, False, HANDLERS[handler])
        if st_ == 4:
            assert res is None
            declined += 1
            continue
        assert st_ == CODE[w.status], (b, st_, w.status)
        assert res == w.result, (b, res, w.result)
    assert declined <= allow_decline * len(payloads), (declined, len(payloads))
    return declined


def test_table(parser):
    for tok, want in TABLE_IDENTITY:
        assert parser.run(_payload_tok(tok), False, 0) == (0, want), tok
    for tok, want in TABLE_SUM:
        assert parser.run(_payload_tok(b'{"values": ' + tok + b"}"), False, 3) == (0, want), tok
    for tok in TABLE_SUM_DECLINED:
        assert parser.run(_payload_tok(b'{"values": ' + tok + b"}"), False, 3) == (4, None), tok
    _check(parser, [_payload_tok(t) for t, _ in TABLE_IDENTITY], "identity")
    _check(parser, [_payload_tok(b'{"values": ' + t + b"}") for t, _ in TABLE_SUM + [(t, None) for t in TABLE_SUM_DECLINED]],
           "json_sum", allow_decline=0.2)


def test_declines_are_the_documented_ones(parser):
    deep = b"[" * 17 + b"1" + b"]" * 17
    wide = b"{" + b", ".join(b'"k%d": %d' % (i, i) for i in range(65)) + b"}"
    long_mid = b"9007199254740993.00000000000000000001"          # > 19 digits just above a midpoint: w and w + 1 disagree
    long_ok = b"1.00000000000000000000001"                       # > 19 digits, far from a rounding boundary
    assert parser.run(_payload_tok(deep), False, 0)[0] == 4
    assert parser.run(_payload_tok(wide), False, 0)[0] == 4
    assert parser.run(_payload_tok(b"[" * 16 + b"1" + b"]" * 16), False, 0)[0] == 0
    assert parser.run(_payload_tok(long_mid), False, 0) == (4, None)
    assert parser.run(_payload_tok(long_ok), False, 0) == (0, b"1")
    assert parser.run(_payload_tok(b'{"values": [9223372036854775807, 1]}'), False, 3)[0] == 4   # beyond a C long
    assert parser.run(_payload_tok(b'{"values": [1e19]}'), False, 3)[0] == 4


json_leaf = (st.none() | st.booleans() | st.integers(-(2 ** 70), 2 ** 70) | st.floats(allow_nan=False, allow_infinity=False)
             | st.text(max_size=6))
json_val = st.recursive(json_leaf, lambda c: st.lists(c, max_size=5) | st.dictionaries(st.text(max_size=3), c, max_size=5),
                        max_leaves=20)


@settings(max_examples=400, deadline=None, suppress_health_check=list(HealthCheck))
@given(st.lists(json_val, min_size=1, max_size=20))
def test_identity_over_python_values(parser, vals):
    _check(parser, [loop.sdk_put_payload(v) for v in vals], "identity")


def _sum_term_in_domain(x: float) -> bool:
    """Go writes an integral float below 1e21 as digits: from 2^63 on, Python's int is beyond a C long (a documented decline)"""
    return not (x == int(x) and 2 ** 63 <= abs(x) < 1e21)


@settings(max_examples=400, deadline=None, suppress_health_check=list(HealthCheck))
@given(st.lists(st.lists(st.floats(allow_nan=False, allow_infinity=False, width=64).filter(_sum_term_in_domain) | st.integers(-(2 ** 58), 2 ** 58)
                         | st.booleans() | st.sampled_from([0.1, 0.2, 0.3, 1e16, -1e16, 1e308, -1e308, 5e-324, -0.0]), max_size=12),
                min_size=1, max_size=20))
def test_json_sum_over_python_floats(parser, lists):
    """pins the restated float summation against the real builtin sum (CPython >= 3.12: Neumaier compensation)"""
    assert sys.version_info >= (3, 12)
    payloads = [loop.sdk_put_payload({"values": v}) for v in lists]
    for v in lists:
        assert not any(isinstance(x, int) and abs(x) > 2 ** 58 for x in v)   # 12 terms stay inside a C long
    _check(parser, payloads, "json_sum")


def test_generated_batches_and_byte_mutants(parser):
    from beta9_b200 import synth
    vb = synth.values_batch(3000, seed=11)
    fb = synth.json_float_batch(600, seed=12)
    assert _check(parser, vb.tasks(), "identity") == 0
    assert _check(parser, fb.tasks(), "json_sum") == 0
    rng = np.random.default_rng(7)
    alphabet = list(b'{}[],:" 0159e.-+Etrue\\')
    muts = []
    for p in vb.tasks()[:600] + fb.tasks()[:200]:
        for _ in range(3):
            m = bytearray(p)
            pos = int(rng.integers(10, len(m) - 17))
            op = int(rng.integers(0, 3))
            ch = int(rng.choice(alphabet))
            if op == 0: m[pos] = ch
            elif op == 1: del m[pos]
            else: m[pos:pos] = bytes([ch])
            muts.append(bytes(m))
    # (mutated numbers can carry > 19 digits at a rounding boundary, or run past a C long: those few may be declined)
    _check(parser, muts, "identity", allow_decline=0.01)
    _check(parser, muts, "json_sum", allow_decline=0.01)
