"""The user-handler header's contract on a CPU: the test-only handlers of tests/handlers (script, script_sig, inspect,
inspect_keys), compiled for the host by tests/host_shim/contract_shim.cpp with include/b9gpu_handler.cuh, against their
Python twins (tests/handlers/contract_twins.py).

script drives every sink call and every broken rule the header names; its twin states what the record must be, and the
runner's own loops (run_task_loop, the runner's half over TaskMessage records, the endpoint request) render the value.
script_sig runs the same scripts through the settle rules of a handler with a signature: both forms must give the same
record. inspect and inspect_keys write what kind / number / empty / chars / items / both get overloads see of an
argument; their twins write the same from the value json.loads gave the runner. Statuses, has_result, exception bits
and record bytes must all agree, and no writing pass may touch a byte past its record's reservation. The corpora are
functions of this module so that tests/test_gpu_handler_contract.py runs the same ones on the device."""
import ctypes as C
import json
import math
import os
import re
import struct

import numpy as np
import pytest

from oracle.pyoracle import endpoint as EP
from oracle.pyoracle.gojson import GoJSONError
from oracle.pyoracle.httpserialize import InvalidRequestPayload
from oracle.pyoracle.loop import run_task_loop
from tests import test_user_handler_on_host as U
from tests.handlers import contract_twins as T
from tests.task_msg_oracle import NOT_RUN, run_records

HERE, ROOT = U.HERE, U.ROOT
SRC = os.path.join(HERE, "host_shim", "contract_shim.cpp")
SO = os.path.join(HERE, "host_shim", "libcontractshim.so")
NAMES = ["script", "script_sig", "inspect", "inspect_keys"]
COMPLETE, ERROR, REJECTED, UNSUPPORTED = U.COMPLETE, U.ERROR, U.REJECTED, U.UNSUPPORTED
TF_HTTP_BODY, TF_TASK_MSG, TQ, ENDPOINT = U.TF_HTTP_BODY, U.TF_TASK_MSG, U.TQ, U.ENDPOINT
# (source, rendering, slot flags): SDK payloads, HTTP bodies and TaskMessage records for the task queue, HTTP bodies for
# the endpoint
SOURCES = [("sdk", TQ, 0), ("http", TQ, TF_HTTP_BODY), ("record", TQ, TF_TASK_MSG), ("endpoint", ENDPOINT, TF_HTTP_BODY)]


@pytest.fixture(scope="module")
def ct():
    lib = U._shim(SRC, SO, ["-I" + os.path.join(ROOT, "include")])
    u64p, u8p, i64p = (np.ctypeslib.ndpointer(t, flags="C") for t in (np.uint64, np.uint8, np.int64))
    lib.b9_ct_batch.argtypes = [C.c_char_p, u64p, u8p, u8p, C.c_uint32, C.c_int, C.c_int, u8p, u8p, i64p, u8p, C.c_void_p, u64p]
    lib.b9_ct_batch.restype = C.c_uint64

    def batch(payloads, name, rendering, flags=0, ids=None):
        """[(status, has, exception bit, record bytes)] per payload"""
        n = len(payloads)
        if not n:
            return []
        off = np.zeros(n + 1, np.uint64)
        np.cumsum([len(b) for b in payloads], out=off[1:])
        blob = b"".join(payloads) + b"\0" * 8
        fl = np.full(n, flags, np.uint8)
        idb = np.frombuffer(b"".join(ids), np.uint8).copy() if ids is not None else np.zeros(n * 16, np.uint8)
        status, has, val, guard = (np.zeros(n, np.uint8), np.zeros(n, np.uint8), np.zeros(n, np.int64), np.zeros(n, np.uint8))
        out_off = np.zeros(n + 1, np.uint64)
        h = NAMES.index(name)
        total = lib.b9_ct_batch(blob, off, fl, idb, n, h, rendering, status, has, val, guard, None, out_off)
        out = np.zeros(total + 1, np.uint8)
        lib.b9_ct_batch(blob, off, fl, idb, n, h, rendering, status, has, val, guard, out.ctypes.data, out_off)
        # the writing sink never writes past the record's reservation
        assert guard.all(), [payloads[i] for i in np.flatnonzero(guard == 0)[:5]]
        raw = out.tobytes()
        return [(int(status[i]), int(has[i]), int(val[i]), raw[int(out_off[i]):int(out_off[i + 1])] if has[i] else b"")
                for i in range(n)]
    return batch


def same(got, want):
    """a record against its expectation; a device record carries no exception class (None)"""
    return got[:2] == want[:2] and got[3] == want[3] and (got[2] is None or got[2] == want[2])


# ---- scripts --------------------------------------------------------------------------------------------------------------
def bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def op(code, v=None):
    """one op; a 64-bit argument goes as two halves"""
    if v is None:
        return [code]
    if code in (T.INT, T.REAL) and not -2**31 <= v < 2**31:
        return [code] + T.halves(v)
    return [code, v]


CPS = [0x41, 0x22, 0x5C, 0x0A, 0x00, 0x1F, 0x7F, 0x80, 0xE9, 0x7FF, 0x800, 0x20AC, 0xFFFF, 0x10000, 0x1F600, 0x10FFFF,
       0xD800, 0xDBFF, 0xDC00, 0xDFFF, 0x110000]
REAL_BITS = [0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0x7FF8DEADBEEF0001, 0xFFF0000000000ABC,
             0x7FF0000000000000, 0xFFF0000000000000, 0, 0x8000000000000000, 1, 0x000FFFFFFFFFFFFF, 0x800FFFFFFFFFFFFF,
             0x0010000000000000, bits(1e16), bits(math.nextafter(1e16, 0)), bits(1e-4), bits(math.nextafter(1e-4, 0)), bits(1e-5),
             bits(1e-7), bits(1.5), bits(-2.5), bits(0.1), bits(1e21), bits(1e22), bits(123.0), bits(1.7976931348623157e308)]
INTS = [T.INT64_MIN, T.INT64_MAX, 0, -1, 1, 2**53 + 1, -(2**53) - 1, 2**32, 2**31 - 1, -(2**31)]
RETURNS = list(range(-2, 0x41))

# the op instances the pair corpus combines: each code, with arguments at their edges
OPS = [op(T.NONE), op(T.BOOL, 0), op(T.BOOL, 1), op(T.BOOL, 2), op(T.INT, 0), op(T.INT, -1), op(T.INT, 7), op(T.INT, T.INT64_MIN),
       op(T.INT, T.INT64_MAX), op(T.REAL, bits(1.5)), op(T.REAL, bits(-0.0)), op(T.REAL, 0), op(T.REAL, 0x7FF8000000000000),
       op(T.REAL, 0xFFF0000000000000), op(T.STR_BEGIN), op(T.CP, 0x41), op(T.CP, 0xE9), op(T.CP, 0x1F600), op(T.CP, 0xD800),
       op(T.CP, 0x110000), op(T.CP, 0x22), op(T.STR_END), op(T.RETURN, 0), op(T.RETURN, 1), op(T.RETURN, 0x20), op(T.RETURN, 3),
       op(T.RETURN, 0x40), op(T.RETURN, -1), op(T.RETURN, -2), op(T.CP_WRITE, 0x41), op(T.CP_WRITE, 0xD800),
       op(T.CP_COUNT, 0x41), op(T.CP_COUNT, 0xE9), op(T.CP_COUNT, 0x800)]


def pair_scripts():
    """every op and every pair of ops, each alone and inside a string ([str_begin] ... [str_end])"""
    out = []
    for a in OPS:
        out += [[a], [op(T.STR_BEGIN), a, op(T.STR_END)]]
        for b in OPS:
            out += [[a, b], [op(T.STR_BEGIN), a, b, op(T.STR_END)]]
    return out


def edge_scripts():
    """every real edge, integer edge and return value, alone and around a written value"""
    s = op(T.STR_BEGIN), op(T.CP, 0x41), op(T.STR_END)
    out = []
    for b in REAL_BITS:
        out += [[op(T.REAL, b)], [op(T.REAL, b), op(T.RETURN, 0)], [op(T.REAL, b), op(T.NONE)]]
    for v in INTS:
        out += [[op(T.INT, v)], [op(T.INT, v), op(T.RETURN, 0)]]
    for r in RETURNS:
        out += [[op(T.RETURN, r)], [*s, op(T.RETURN, r)], [op(T.NONE), op(T.NONE), op(T.RETURN, r)], [op(T.STR_BEGIN), op(T.RETURN, r)]]
    out += [[], [op(T.RETURN, 0), [99]], [[99]], [[]], [[1, 2, 3, 4]], [[0.5]], [[True]], [op(T.STR_BEGIN), [T.CP, 0.5]]]
    out += [[op(T.STR_BEGIN)] + [op(T.CP, c) for c in CPS if T._cp_ok(c)] + [op(T.STR_END)]]
    return out


def _cp_pool(rng):
    k = int(rng.integers(0, 8))
    lo_hi = [(0, 0x80), (0x80, 0x800), (0x800, 0xD800), (0xE000, 0x10000), (0x10000, 0x110000), (0xD800, 0xE000)]
    if k < len(lo_hi):
        return int(rng.integers(*lo_hi[k]))
    if k == 6:
        return int(rng.choice([0x10FFFF, 0x110000, 0xFFFFFFFF]))
    return int(rng.choice([0x22, 0x5C, 0x08, 0x0C, 0x0A, 0x0D, 0x09, 0x00, 0x1F, 0x7F, 0x2F, 0x2028]))


def random_scripts(n, seed):
    """n random scripts of up to 12 ops: mostly strings of code points from every UTF-8 length, surrogates, U+10FFFF and
    beyond, and what json.dumps escapes, with now and then an op of another kind, a pass-only code point or a return"""
    rng = np.random.default_rng(seed)
    pool_bits = REAL_BITS + [int(x) for x in rng.integers(0, 2**64, size=64, dtype=np.uint64)]
    out = []
    for _ in range(n):
        ops = []
        for _ in range(int(rng.integers(0, 13))):
            r = rng.random()
            if r < 0.55:
                ops.append(op(int(rng.choice([T.CP, T.CP, T.CP, T.CP_WRITE, T.CP_COUNT])), _cp_pool(rng)))
            elif r < 0.62:
                ops.append(op(T.STR_BEGIN))
            elif r < 0.69:
                ops.append(op(T.STR_END))
            else:
                code = int(rng.integers(0, 8))
                v = {T.BOOL: int(rng.integers(0, 3)), T.INT: INTS[int(rng.integers(0, len(INTS)))],
                     T.REAL: pool_bits[int(rng.integers(0, len(pool_bits)))], T.RETURN: RETURNS[int(rng.integers(0, len(RETURNS)))] if rng.random() < 0.5 else 0,
                     T.CP: _cp_pool(rng)}.get(code)
                ops.append(op(code, v))
        if rng.random() < 0.6:                                  # a string around them
            ops = [op(T.STR_BEGIN)] + ops + [op(T.STR_END)]
        out.append(ops)
    return out


def sources_of(payloads):
    """[(source, rendering, flags, payloads, ids)]: the same calls as each source carries them"""
    recs, ids = U.records_of(payloads)
    out = []
    for source, rendering, flags in SOURCES:
        if source == "record":
            out.append((source, rendering, flags, recs, ids))
        else:
            out.append((source, rendering, flags, list(payloads), None))
    return out


def sdk(*args, **kwargs):
    return json.dumps({"args": list(args), "kwargs": kwargs}).encode()


def expected(fn, source, rendering, payloads, ids, outcome):
    """the records the runner makes of `payloads` with handler `fn`; outcome(args, kwargs) says where the device must
    decline (UNSUPPORTED) and returns the exception bit a raising call raises"""
    out = []
    if rendering == ENDPOINT:
        for p in payloads:
            try:
                fwd = json.loads(EP.gateway_body(p))
            except (InvalidRequestPayload, GoJSONError, ValueError, RecursionError):
                fwd = None
            oc, body = EP.run_endpoint_request(p, fn)
            kind, bit = outcome(fwd["args"] or [], fwd["kwargs"] or {}) if fwd is not None else (None, 0)
            if kind == T.UNSUPPORTED:
                out.append((UNSUPPORTED, 0, 0, b""))
            elif oc == EP.BAD_REQUEST:
                out.append((REJECTED, 0, 0, b""))
            elif oc == EP.HANDLER_RAISED:
                out.append((ERROR, 0, bit, b""))
            else:
                assert oc == EP.OK, (p, oc)
                out.append((COMPLETE, 1, 0, body))
        return out
    if source == "record":
        want = run_records(payloads, ids, fn)
    else:
        want = run_task_loop(payloads, [i.to_bytes(16, "little") for i in range(len(payloads))], handler=fn,
                             http_body=source == "http", keep_wire=True)
    for w in want:
        assert w.status != NOT_RUN
        if w.status == "REJECTED":
            out.append((REJECTED, 0, 0, b""))
            continue
        t = json.loads(w.wire)
        kind, bit = outcome(t["args"] or [], t["kwargs"] or {})
        if kind == T.UNSUPPORTED:
            out.append((UNSUPPORTED, 0, 0, b""))
        elif w.status == "ERROR":
            out.append((ERROR, 0, bit, b""))
        else:
            out.append((COMPLETE, 1 if w.result is not None else 0, 0, w.result or b""))
    return out


def script_outcome(rendering):
    def outcome(args, kwargs):
        kind, x = T.expect(args[0], rendering)
        return kind, x if kind == T.ERROR else 0
    return outcome


def check_scripts(run, scripts):
    """every script from every source, under both handler forms, against expect and the runner's rendering; both forms
    must give the same records (the two copies of the settle rules agree)"""
    payloads = [sdk(s) for s in scripts]
    for source, rendering, flags, ps, ids in sources_of(payloads):
        want = expected(T.twin(rendering), source, rendering, ps, ids, script_outcome(rendering))
        by_form = {}
        for name in ("script", "script_sig"):
            got = run(ps, name, rendering, flags, ids)
            for s, g, w in zip(scripts, got, want):
                assert same(g, w), (name, source, s, g, w)
            by_form[name] = [(g[0], g[1], g[3]) for g in got]
        assert by_form["script"] == by_form["script_sig"]


# ---- inspect ---------------------------------------------------------------------------------------------------------------
_NUM = re.compile(rb"-?[0-9][0-9.]*(?:[eE][-+]?[0-9]+)?")


def _over_19_digits(payload):
    """a number literal of more than 19 significant digits: f64_parse may not settle it"""
    for m in _NUM.findall(payload):
        mant = re.split(rb"[eE]", m.lstrip(b"-"))[0].replace(b".", b"").lstrip(b"0").rstrip(b"0")
        if len(mant) > 19:
            return True
    return False


def _too_deep(payload):
    return payload.count(b"[") + payload.count(b"{") > 60


def inspect_outcome(fn):
    def outcome(args, kwargs):
        try:
            fn(*args, **kwargs)
        except T.Unsure:
            return T.UNSUPPORTED, 0                         # number() cannot answer: the record is UNSUPPORTED
        except TypeError:
            return T.ERROR, 0x01
        return T.VALUE, 0
    return outcome


def _declining(fn):
    def f(*args, **kwargs):
        try:
            return fn(*args, **kwargs)
        except T.Unsure:
            raise T.Declined() from None
    return f


def check_inspect(run, name, payloads, min_share=0.9):
    """inspect / inspect_keys over payloads from every source; an UNSUPPORTED the twin does not predict must be one of
    the documented reasons: a literal of more than 19 significant digits or nesting past the parser's limit"""
    fn = {"inspect": T.inspect, "inspect_keys": T.inspect_keys}[name]
    for source, rendering, flags, ps, ids in sources_of(payloads):
        want = expected(_declining(fn), source, rendering, ps, ids, inspect_outcome(fn))
        got = run(ps, name, rendering, flags, ids)
        answered = 0
        for p, g, w in zip(ps, got, want):
            if g[0] == UNSUPPORTED and w[0] != UNSUPPORTED:
                assert _over_19_digits(p) or _too_deep(p), (name, source, p, w)
                continue
            answered += 1
            assert same(g, w), (name, source, p, g, w)
        assert answered >= min_share * len(ps), (name, source, answered, len(ps))


KEY_SPELLINGS = [
    '{"a": 1}', '{"\\u0061": 1}', '{"a": 1, "a": 2}', '{"a": 1, "\\u0061": 2}', '{"\\u0061": 1, "a": [2, 3]}',
    '{"values": [1, 2.5, "x"]}', '{"valu\\u0065s": {"a": null}}', '{"\\u00e9": 1}', '{"\xc3\xa9": 2}', '{"\\u00E9": 3, "\xc3\xa9": 4}',
    '{"\\u20ac": 1}', '{"\xe2\x82\xac": true}', '{"\\ud83d\\ude00": 1}', '{"\xf0\x9f\x98\x80": "s"}', '{"\\uD83D\\uDE00": 1, "\xf0\x9f\x98\x80": 2}',
    '{"": 0}', '{"": 1, "": 2}', '{"a\\"b": 1}', '{"a\\u0022b": [1]}', '{"a\\"b": 1, "a\\u0022b": 2}', '{"\\ud83d": 1}',
    '{"\\ude00": 1, "\\ud83d": 2}', '{"e\\u0301": 1}', '{"A": 1}', '{"a ": 1}', '{"a\\u0000": 1}', '{"\\u0061\\u0022\\u0062": 5}',
    '{"values": 1, "a": 2, "\\u00e9": 3, "\\u20ac": 4, "\\ud83d\\ude00": 5, "": 6, "a\\"b": 7}',
    '{"a": {"a": {"a": {"a": 1}}}}', '{"values": [[[[1]]]]}', '{"a": [{"values": [{"a": 1}]}]}',
    '{"a": 1e20, "values": 1e21, "\\u00e9": -0, "\\u20ac": 0.0, "": -0.0, "a\\"b": 1E2}',
    '{"a": 9223372036854775807, "values": -9223372036854775808, "\\u00e9": 9223372036854775808}',
    '{"a": 12345678901234567890123, "values": 1}', '{"values": 1, "zz": 12345678901234567890123}',
]


def key_payloads():
    """dicts whose keys are spelled with escapes, raw UTF-8, surrogate pairs, lone surrogates and duplicates"""
    return [('{"args": [%s], "kwargs": {}}' % d).encode("latin-1") for d in KEY_SPELLINGS]


def value_payloads():
    """the f64 literal and value-edge corpora, the pickle-free value corpora, the user-handler corpus"""
    from tests import pickle_corpus
    from tests.f64_corpus import _literals, value_edge_payloads
    rng = np.random.default_rng(17)
    lits = _literals()
    pick = [lits[i] for i in rng.choice(len(lits), 3000, replace=False)] + ["1e20", "1e21", "-0", "0.0", "-0.0", "1E2",
                                                                            "9223372036854775807", "9223372036854775808",
                                                                            "-9223372036854775808", "-9223372036854775809"]
    out = [('{"args": [%s], "kwargs": {}}' % s).encode() for s in pick]
    out += [('{"args": [[%s, true, false, null, "%s"]], "kwargs": {}}' % (s, s)).encode() for s in pick[:500]]
    out += [p for p, _ in value_edge_payloads() if len(p) < 70000]
    vals = pickle_corpus.plain_values() + pickle_corpus.json_sum_values()
    for v in vals:
        try:
            out.append(json.dumps({"args": [v], "kwargs": {}}).encode())
        except (TypeError, ValueError):
            pass
    return list(dict.fromkeys(out + U.HANDMADE + key_payloads()))


def inspect_keys_payloads():
    ds = [{"a": 1, "values": [1, 2], "é": "x", "€": None, "\U0001F600": 1.5, "": True, 'a"b': {"a": 0}, "b": -0.0}, {}, {"a": 2}]
    keys = T.PROBES + ["b", "A", "é", "\U0001F601", "valuesx", "", "\ud83d"]
    out = [sdk(d, *keys) for d in ds] + [sdk(d) for d in ds] + [sdk(d, k) for d in ds for k in keys]
    out += [sdk([1], "a"), sdk("a", "a"), sdk(None, "a"), sdk(ds[0], 1, None, ["a"], {"a": 1}, True), sdk()]
    for body in KEY_SPELLINGS:                                    # the raw spellings, keys passed escaped and raw
        for k in ('"a"', '"\\u0061"', '"\\u00e9"', '"\xc3\xa9"', '"\\u20ac"', '"\\ud83d\\ude00"', '"\xf0\x9f\x98\x80"', '""',
                  '"a\\"b"', '"a\\u0022b"', '"\\ud83d"', '"values"', '"zz"'):
            out.append(('{"args": [%s, %s, "a"], "kwargs": {}}' % (body, k)).encode("latin-1"))
    out.append(b'{"args": [], "kwargs": {"d": {"a": 1}}}')
    out.append(b'{"args": [{"a": 1}], "kwargs": {"d": 2}}')
    return out


# ---- tests -------------------------------------------------------------------------------------------------------------------
def test_every_op_and_pair_of_ops(ct):
    check_scripts(ct, pair_scripts())


def test_reals_integers_and_return_values(ct):
    check_scripts(ct, edge_scripts())


def test_random_scripts(ct):
    check_scripts(ct, random_scripts(3000, 7))


def test_broken_rules_are_unsupported(ct):
    """each broken rule the header names makes the record UNSUPPORTED, in both renderings and both forms"""
    s, e, a = op(T.STR_BEGIN), op(T.STR_END), op(T.CP, 0x41)
    broken = {
        "a second value": [[op(T.INT, 1), op(T.INT, 2)], [op(T.NONE), op(T.BOOL, 1)], [s, e, op(T.NONE)], [op(T.REAL, 0), s, e]],
        "a string left open": [[s], [s, a]],
        "cp outside a string": [[a], [s, e, a], [op(T.CP, 0x41), s, e]],
        "a surrogate or past U+10FFFF": [[s, op(T.CP, c), e] for c in (0xD800, 0xDBFF, 0xDC00, 0xDFFF, 0x110000, 0xFFFFFFFF)],
        "no value": [[], [op(T.RETURN, 0)]],
        "a return of two bits, 0x40 or -2": [[op(T.RETURN, r)] for r in (3, 0x21, 0x3F, 0x40, 0x80, -2)] + [[s, a, e, op(T.RETURN, 3)]],
        "a declined task": [[op(T.RETURN, -1)], [s, a, e, op(T.RETURN, -1)]],
        "a writing pass longer than counted": [[s, a, op(T.CP_WRITE, 0x41), e], [s, a, op(T.CP_WRITE, 0xE9), e],
                                               [s, a, op(T.CP_WRITE, 0x1F600), e]],
        "a writing pass shorter than counted": [[s, a, op(T.CP_COUNT, 0x41), e], [s, op(T.CP_COUNT, 0x20AC), a, e]],
        "the same length, a surrogate written": [[s, op(T.CP_COUNT, 0xE9), op(T.CP_WRITE, 0xD800), e],
                                                 [s, op(T.CP_COUNT, 0x800), op(T.CP_WRITE, 0xDC00), e]],
    }
    for rule, scripts in broken.items():
        for ops in scripts:
            for rendering in (TQ, ENDPOINT):
                if rule == "the same length, a surrogate written" and (ops[1][1] == 0xE9) != (rendering == TQ):
                    continue                                      # (the lengths match in one rendering only)
                assert T.expect(ops, rendering) == (T.UNSUPPORTED, None), (rule, ops)
                for name in ("script", "script_sig"):
                    g = ct([sdk(ops)], name, rendering, TF_HTTP_BODY)[0]
                    assert g == (UNSUPPORTED, 0, 0, b""), (rule, ops, name, rendering, g)


def test_each_exception_class(ct):
    """a single B9_EXC_* bit raises that class (binascii.Error included): ERROR with the bit, in both forms and renderings"""
    for bit, cls in T.EXC_CLASSES.items():
        assert type(T.exception(bit)) is cls
        for name in ("script", "script_sig"):
            for rendering in (TQ, ENDPOINT):
                g = ct([sdk([op(T.RETURN, bit)]), sdk([op(T.INT, 5), op(T.RETURN, bit)])], name, rendering, TF_HTTP_BODY)
                assert g == [(ERROR, 0, bit, b"")] * 2, (bit, name, rendering, g)


def test_scalars_in_both_renderings(ct):
    """None, bools, ints, NaN, infinities, -0.0 and subnormals as the runner renders them, spelled out"""
    cases = [([op(T.NONE)], None, b"null"), ([op(T.BOOL, 1)], b"true", b"true"), ([op(T.BOOL, 0)], None, b"false"),
             ([op(T.INT, T.INT64_MIN)], b"-9223372036854775808", b"-9223372036854775808"), ([op(T.INT, 0)], None, b"0"),
             ([op(T.REAL, 0xFFF8000000000001)], b"NaN", UNSUPPORTED), ([op(T.REAL, 0x7FF0000000000000)], b"Infinity", UNSUPPORTED),
             ([op(T.REAL, 0xFFF0000000000000)], b"-Infinity", UNSUPPORTED), ([op(T.REAL, 0x8000000000000000)], None, b"-0.0"),
             ([op(T.REAL, 1)], b"5e-324", b"5e-324"), ([op(T.REAL, bits(1e16))], b"1e+16", b"1e+16"),
             ([op(T.REAL, bits(1e-5))], b"1e-05", b"1e-05"), ([op(T.REAL, bits(1e-4))], b"0.0001", b"0.0001"),
             ([op(T.STR_BEGIN), op(T.STR_END)], None, b'""'),
             ([op(T.STR_BEGIN), op(T.CP, 0xE9), op(T.CP, 0x1F600), op(T.CP, 0x0A), op(T.STR_END)], b'"\\u00e9\\ud83d\\ude00\\n"',
              '"é\U0001F600\\n"'.encode())]
    for ops, tq, ep in cases:
        g = ct([sdk(ops)], "script", TQ)[0]
        assert g == ((COMPLETE, 1, 0, tq) if tq is not None else (COMPLETE, 0, 0, b"")), (ops, g)
        g = ct([sdk(ops)], "script", ENDPOINT, TF_HTTP_BODY)[0]
        assert g == ((UNSUPPORTED, 0, 0, b"") if ep == UNSUPPORTED else (COMPLETE, 1, 0, ep)), (ops, g)


def test_script_sig_binds_its_call(ct):
    """script_sig(ops, *rest) by keyword and with surplus positionals; script(ops, /) refuses both"""
    ops = [op(T.INT, 3)]
    for body in (sdk(ops, 1, "x"), json.dumps({"args": [], "kwargs": {"ops": ops}}).encode()):
        assert ct([body], "script_sig", TQ)[0] == (COMPLETE, 1, 0, b"3")
        assert ct([body], "script", TQ)[0] == (ERROR, 0, 0x01, b"")


def test_inspect_values(ct):
    check_inspect(ct, "inspect", value_payloads())


def test_inspect_key_spellings(ct):
    check_inspect(ct, "inspect", key_payloads(), min_share=0.8)
    # (the last of duplicate keys wins; an escaped key equals its raw spelling)
    g = ct([b'{"args": [{"a": 1, "\\u0061": 2, "\\u00e9": [3], "\xc3\xa9": 4}], "kwargs": {}}'], "inspect", TQ)[0]
    assert g[3] == b'"D0{I0=i2,-,I0=i4,-,-,-,-}"', g


def test_inspect_keys(ct):
    check_inspect(ct, "inspect_keys", inspect_keys_payloads(), min_share=0.8)


def test_unsure_numbers_are_unsupported(ct):
    """number() on an int past int64 (or a literal f64_parse cannot settle) makes the record UNSUPPORTED, whatever the
    handler writes; an int64 edge is answered"""
    for lit in ("9223372036854775808", "-9223372036854775809", "1e19", "18446744073709551616", "99999999999999999999"):
        for rendering, fl in ((TQ, 0), (ENDPOINT, TF_HTTP_BODY)):
            assert ct([('{"args": [%s]}' % lit).encode()], "inspect", rendering, fl)[0] == (UNSUPPORTED, 0, 0, b""), lit
    # (Go writes the float64 of -2**63 as -9223372036854776000, past int64; the largest magnitude Go's text keeps in it:)
    assert ct([b'{"args": [-9223372036854775000]}'], "inspect", TQ)[0][3] == b'"I0=i-9223372036854775000"'
    # an unsure number the handler never asks about does not matter
    assert ct([b'{"args": [{"zz": 12345678901234567890123}]}'], "inspect", TQ)[0][0] == COMPLETE
