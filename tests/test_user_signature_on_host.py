"""User handlers with a declared signature on a CPU: the signature half of the user-handler drain (include/b9gpu_handler.cuh:
where a call's positional and keyword arguments are in an SDK payload, an HTTP body or a TaskMessage record, CPython's
binding of handler(*args, **kwargs), phase A and B around the bound call) and the example handlers that declare one
(greet, join, field_sum in examples/handlers), compiled for the host by tests/host_shim/user_signature_shim.cpp, against
their Python twins run through the oracle's loops, which call fn(*args, **kwargs): CPython is the reference for binding.
Statuses, has_result, record bytes and the exception class of every ERROR must agree; an UNSUPPORTED must carry one of
the documented reasons (`may_decline`). `probe` (in the shim) covers every parameter kind. The compile-time checks of
B9H_SIGNATURE are tested with g++ and nvcc."""
import ctypes as C
import inspect
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from oracle.pyoracle import endpoint as EP
from oracle.pyoracle.httpserialize import InvalidRequestPayload
from oracle.pyoracle.gojson import GoJSONError
from oracle.pyoracle.loop import run_task_loop
from tests import test_user_handler_on_host as U
from tests.task_msg_oracle import NOT_RUN, run_records

twins = U.twins
HERE, ROOT = U.HERE, U.ROOT
SRC = os.path.join(HERE, "host_shim", "user_signature_shim.cpp")
SO = os.path.join(HERE, "host_shim", "libusersignatureshim.so")
NAMES = ["greet", "join", "field_sum", "probe"]
COMPLETE, ERROR, REJECTED, UNSUPPORTED = U.COMPLETE, U.ERROR, U.REJECTED, U.UNSUPPORTED
TF_HTTP_BODY, TF_TASK_MSG, TQ, ENDPOINT = U.TF_HTTP_BODY, U.TF_TASK_MSG, U.TQ, U.ENDPOINT
_UNSET = object()


def probe(a, /, b, c=_UNSET, *rest, d, e=_UNSET):
    def tag(v):
        return "-" if v is _UNSET else v if type(v) is str else type(v).__name__
    return "|".join(tag(v) for v in (a, b, c, d, e) + rest)


FNS = {"greet": twins.greet, "join": twins.join, "field_sum": twins.field_sum, "probe": probe}


@pytest.fixture(scope="module")
def us():
    lib = U._shim(SRC, SO, ["-I" + os.path.join(ROOT, "include")])
    u64p, u8p, i64p = (np.ctypeslib.ndpointer(t, flags="C") for t in (np.uint64, np.uint8, np.int64))
    lib.b9_us_batch.argtypes = [C.c_char_p, u64p, u8p, u8p, C.c_uint32, C.c_int, C.c_int, u8p, u8p, i64p, C.c_void_p, u64p]
    lib.b9_us_batch.restype = C.c_uint64

    def batch(payloads, name, rendering, flags=0, ids=None):
        """[(status, has, exception bit, record bytes)] per payload"""
        n = len(payloads)
        off = np.zeros(n + 1, np.uint64)
        np.cumsum([len(b) for b in payloads], out=off[1:])
        blob = b"".join(payloads) + b"\0" * 8
        fl = np.full(max(n, 1), flags, np.uint8)
        idb = np.frombuffer(b"".join(ids), np.uint8).copy() if ids is not None else np.zeros(max(n, 1) * 16, np.uint8)
        status, has, val = np.zeros(max(n, 1), np.uint8), np.zeros(max(n, 1), np.uint8), np.zeros(max(n, 1), np.int64)
        out_off = np.zeros(n + 1, np.uint64)
        h = NAMES.index(name)
        total = lib.b9_us_batch(blob, off, fl, idb, n, h, rendering, status, has, val, None, out_off)
        out = np.zeros(total + 1, np.uint8)
        lib.b9_us_batch(blob, off, fl, idb, n, h, rendering, status, has, val, out.ctypes.data, out_off)
        raw = out.tobytes()
        return [(int(status[i]), int(has[i]), int(val[i]), raw[int(out_off[i]):int(out_off[i + 1])]) for i in range(n)]
    return batch


# ---- when may the device decline? -------------------------------------------------------------------------------------
_FOLD = str.maketrans({"K": "k", "ſ": "s"})


def _kwargs_merged(payload: bytes) -> bool:
    """an SDK payload whose "kwargs" (Go's struct keys fold case) came as an object twice without a null between: Go
    merges the maps, which the device does not do"""
    try:
        pairs = json.loads(payload.decode("utf-8", "replace"), object_pairs_hook=lambda kv: kv)
    except (ValueError, RecursionError):
        return False
    if not isinstance(pairs, list):
        return False
    objs = 0
    for k, v in pairs:
        if k.translate(_FOLD).lower() == "kwargs":
            objs = objs + 1 if isinstance(v, list) else 0
    return objs > 1


def _field_sum_overflows(args, kwargs) -> bool:
    """field_sum meets an int outside int64, or its int sum leaves int64 (Python goes on with a big int)"""
    try:
        ba = inspect.signature(twins.field_sum).bind(*args, **kwargs)
    except TypeError:
        return False
    rows, field = ba.arguments["rows"], ba.arguments["field"]
    if type(field) is not str or not isinstance(rows, list):
        return False
    total = 0
    for row in rows:
        if type(row) is not dict or field not in row or type(row[field]) not in (int, float, bool):
            return False
        v = row[field]
        if type(v) is int and not -2**63 <= v < 2**63:
            return True
        total += v
        if type(total) is int and not -2**63 <= total < 2**63:
            return True
    return False


def may_decline(name, payload, args, kwargs, sdk=False):
    if U._long_literal(payload) or (sdk and _kwargs_merged(payload)):
        return True
    return name == "field_sum" and args is not None and _field_sum_overflows(args, kwargs or {})


def exc_bit(fn, args, kwargs):
    try:
        fn(*args, **kwargs)
    except BaseException as e:              # noqa: BLE001
        return U.EXC.get(type(e), -1)
    return 0


# ---- the comparisons ---------------------------------------------------------------------------------------------------
def check_tq(us, name, payloads, http=False):
    """the task-queue rendering against run_task_loop; returns the number of tasks the device answered"""
    fn = FNS[name]
    ids = [i.to_bytes(16, "little") for i in range(len(payloads))]
    want = run_task_loop(payloads, ids, handler=fn, http_body=http, keep_wire=True)
    got = us(payloads, name, TQ, TF_HTTP_BODY if http else 0)
    answered = 0
    for p, w, (st_, has, val, data) in zip(payloads, want, got):
        args = kwargs = None
        if w.wire is not None:
            t = json.loads(w.wire)
            args, kwargs = t["args"] or [], t["kwargs"] or {}
        if st_ == UNSUPPORTED:
            assert may_decline(name, p, args, kwargs, sdk=not http), (name, p, w)
            continue
        answered += 1
        assert st_ == {"COMPLETE": COMPLETE, "ERROR": ERROR, "REJECTED": REJECTED}[w.status], (name, p, w, st_)
        if st_ == COMPLETE:
            assert (has, data if has else None) == (1 if w.result is not None else 0, w.result), (name, p, w.result, data)
        else:
            assert has == 0 and data == b""
        if st_ == ERROR and val is not None:          # (a device drain's records carry no class: None)
            assert val == exc_bit(fn, args, kwargs), (name, p, val)
    return answered


def check_ep(us, name, bodies):
    fn = FNS[name]
    got = us(bodies, name, ENDPOINT, TF_HTTP_BODY)
    answered = 0
    for b, (st_, has, val, data) in zip(bodies, got):
        outcome, want = EP.run_endpoint_request(b, fn)
        fwd = None
        try:
            fwd = json.loads(EP.gateway_body(b))
        except (InvalidRequestPayload, GoJSONError, ValueError, RecursionError):
            pass
        if st_ == UNSUPPORTED:
            assert outcome == EP.RENDER_FAILED or may_decline(name, b, fwd and (fwd["args"] or []), fwd and (fwd["kwargs"] or {})), \
                (name, b, outcome)
            continue
        answered += 1
        if st_ == COMPLETE:
            assert (outcome, data) == (EP.OK, want) and has == 1, (name, b, outcome, want, data)
        elif st_ == REJECTED:
            assert outcome == EP.BAD_REQUEST and has == 0, (name, b, outcome)
        else:
            assert st_ == ERROR and outcome == EP.HANDLER_RAISED and has == 0, (name, b, outcome, st_)
            if val is not None:
                assert val == exc_bit(fn, fwd["args"] or [], fwd["kwargs"] or {}), (name, b, val)
    return answered


def check_records(us, name, records, ids):
    fn = FNS[name]
    want = run_records(records, ids, fn)
    got = us(records, name, TQ, TF_TASK_MSG, ids)
    answered = 0
    for r, w, (st_, has, val, data) in zip(records, want, got):
        t = json.loads(r) if w.status != NOT_RUN else None
        args, kwargs = (t["args"] or [], t["kwargs"] or {}) if t else (None, None)
        if st_ == UNSUPPORTED:
            assert w.status == NOT_RUN or may_decline(name, r, args, kwargs), (name, r, w)
            continue
        answered += 1
        assert st_ == {"COMPLETE": COMPLETE, "ERROR": ERROR}[w.status], (name, r, w)
        assert (has, data if has else None) == (1 if w.result is not None else 0, w.result), (name, r, w.result, data)
        if st_ == ERROR and val is not None:
            assert val == exc_bit(fn, args, kwargs), (name, r, val)
    return answered


def check_all(us, name, payloads, min_share=0.0):
    """SDK payloads, HTTP bodies, TaskMessage records and endpoint requests of the same bytes"""
    n = len(payloads)
    a = check_tq(us, name, payloads)
    b = check_tq(us, name, payloads, http=True)
    c = check_ep(us, name, payloads)
    recs, ids = U.records_of(payloads)
    d = check_records(us, name, recs, ids)
    assert min(a, b, c) >= min_share * n and d >= min_share * len(recs), (name, a, b, c, d, n, len(recs))


# ---- corpora -------------------------------------------------------------------------------------------------------------
def call(*args, **kwargs):
    return args, kwargs


CALLS = {
    "greet": [call(), call("a"), call("a", "b"), call("a", "b", "c"), call(name="x"), call(greeting="x"), call("a", name="b"),
              call("a", bogus=1), call("a", punct="?"), call("a", "hi", punct="?"), call(name="n", greeting="g", punct="p"),
              call("a", context=1), call("a", callback_url="http://x"), call("a", **{"": 1}), call("a", **{"é": 1}),
              call("a", 1), call(1), call("a", punct=None), call("é\U0001F600", "\x00\"\\"), call("", ""),
              call("a", greeting="b"), call("a", "b", greeting="c"), call("a", "b", punct="c", greeting="d"), call(["a"]),
              call(name="a", punct="?", extra=None), call("a", Punct="?"), call("a", "b", "c", punct="?")],
    "join": [call(), call("-"), call("-", "a"), call("-", "a", "b", "c"), call("-", "a", 1), call(sep="-"), call("-", parts=["a"]),
             call(1, "a"), call("", "", ""), call(sep="-", parts="x"), call("é", "\U0001F600", "x"), call("-", "a", sep="-"),
             call("-", "a", context=None), call(", ", *"abcdefghij"), call("-", None), call(None)],
    "field_sum": [call([{"x": 1}], field="x"), call([{"x": 1}]), call([{"x": 1}], "x"), call(rows=[{"x": 1}], field="x"),
                  call([{"x": 1}, {"y": 2}], field="x"), call([{"x": 1.5}, {"x": 2}], field="x"), call([1], field="x"),
                  call([{"x": "a"}], field="x"), call([{"x": 2**62}, {"x": 2**62}], field="x"), call([], field="x"),
                  call("", field="x"), call({}, field="x"), call("ab", field="x"), call({"a": 1}, field="x"),
                  call([{"x": 1}], field=1), call([{"x": True}, {"x": 2}], field="x"), call([{"x": 0.1}, {"x": 0.2}, {"x": 0.3}], field="x"),
                  call([{"x": 1e308}, {"x": 1e308}], field="x"), call([{"x": 2**63 - 1}, {"x": 0.5}], field="x"),
                  call([{"é": 3}, {"é": 4}], field="é"), call([{"x": None}], field="x"), call([{"x": [1]}], field="x"),
                  call(None, field="x"), call(7, field="x"), call([{"x": 1}], field="x", other=1), call(field="x"),
                  call([{"x": -0.0}], field="x"), call([{"x": 1}, {"x": -1}], field="x"), call([{"x": 3}, 5], field="y"),
                  call([{"": 3}], field=""), call([{"x": 1}], field=["x"])],
    "probe": [call(1, 2, d=3), call(1, 2, 3, d=4), call(1, 2, 3, 4, 5, d="d"), call(1, b=2, d=3), call(a=1, b=2, d=3),
              call(1, 2, d=3, e=4), call(1, 2, 3, c=1, d=1), call(1, 2), call(1, d=3), call(), call("s", [1], {"k": 1}, None, True, 1.5, d=0),
              call(1, 2, c="c", d="d", e="e"), call(1, 2, d=3, f=4), call(1, 2, rest=[1], d=3), call(1, 2, d=3, context=0),
              call(1, 2, d=3, callback_url="u"), call("a", "b", "c", "d", "e", "f", "g", "h", "i", d="j", e="k")],
}


def sdk(args, kwargs):
    return json.dumps({"args": list(args), "kwargs": kwargs}).encode()


def renderings(args, kwargs):
    """one call as the bodies a client might send: the SDK's payload, and for HTTP its body with the kwargs as top-level
    keys"""
    out = [sdk(args, kwargs), json.dumps({"args": list(args), "kwargs": kwargs}, ensure_ascii=False).encode()]
    if "args" not in kwargs and "kwargs" not in kwargs:
        out.append(json.dumps(dict({"args": list(args)} if args else {}, **kwargs)).encode())
    return out


RAW = [
    b'{"n\\u0061me": "x"}', b'{"name": "a", "name": "b"}', b'{"name": "a", "n\\u0061me": "b"}', b'{"ARGS": ["x"], "KwArgs": {"punct": "?"}}',
    b'{"\\u0041rgs": ["x"]}', b'{"args": "x", "name": "y"}', b'{"kwargs": 5, "name": "y"}', b'{"kwargs": {"name": "a"}, "punct": "?"}',
    b'{"args": ["a"], "args": 5}', b'{"args": 5, "args": ["a"]}', b'{"kwargs": {"name": "a"}, "kwargs": {"punct": "?"}}',
    b'{"kwargs": {"name": "a"}, "kwargs": null, "kwargs": {"name": "b"}}', b'{"kwargs": {}, "kwargs": {"name": "b"}}',
    b'{"args": ["a"], "kwargs": {"callback_url": "u"}}', b'{"name": "x", "context": 1}', b'{"": 1}', b'{"\\u00e9": 1}',
    b'{"name": "x", "\\ud800": 1}', b'{"name": "x", "nam\xff": 1}', b'{"nam\xff": "x"}', b'{"args": ["a"], "kwargs": null}',
    b'{"args": null, "kwargs": {"name": "z"}}', b"{}", b"", b"null", b" \n", b'{"Name": "x"}', b'{"name": "x", "\\u212a": 1}',
    b'{"args": ["a"], "name": "b"}', b'{"args": ["a"], "punct": "?", "greeting": "g"}', b'{"args": [], "kwargs": {"name": "a"}, "x": 1}',
    b'{"args": [[{"x": 1, "x": 2}]], "kwargs": {"field": "x"}}', b'{"args": [[{"\\u0078": 5}]], "kwargs": {"field": "x"}}',
    b'{"args": [[{"x": 1}, {"x": 2, "\\u0078": 7}]], "kwargs": {"field": "\\u0078"}}', b'{"rows": [{"\xc3\xa9": 2}], "field": "\\u00e9"}',
    b'{"rows": [{"a\xffb": 2}], "field": "a\\ufffdb"}', b'{"rows": [{"\\ud800": 2}], "field": "\\ufffd"}', b'{"rows": [], "field": "x"}',
    b'{"rows": [{"x": 1}], "field": "x", "field": "y"}', b'{"args": [[{"x": 1}]], "field": "x"}', b'{"args": ["-"], "parts": ["a"]}',
    b'{"args": ["-", "a", "b"], "kwargs": {}}', b'{"sep": "-"}', b'{"args": [1, 2], "d": 3}', b'{"args": [1], "b": 2, "d": 3, "e": 4}',
    b'{"a": 1, "b": 2, "d": 3}', b'{"args": [1, 2, 3], "c": 4, "d": 5}', b'{"args": [1, 2, 3, 4], "d": 5, "e": 6}',
    b'{"args": [1, 2], "kwargs": {"d": 3}, "e": 4}', b'{"args": [1, 2], "d": 3, "D": 4}', b'{"args": ["n"], "kwargs": {"punct": "\\ud83d\\ude00"}}',
    b'{"args" : [ "x" ] , "kwargs" : { "punct" : "?" , "greeting" : "yo" } }', b'{"args": [1e400], "name": "x"}', b'{"name": 1e400}',
    b'{"args": ["a"], "kwargs": {"punct": 12345678901234567890123}}', b'{"rows": [{"x": 12345678901234567890}], "field": "x"}',
    b'{"rows": [{"x": 1e20}, {"x": 1}], "field": "x"}', b'{"rows": [{"x": 1E2}, {"x": 1.0}], "field": "x"}',
]


def corpus():
    out = []
    for calls in CALLS.values():
        for args, kwargs in calls:
            out += renderings(args, kwargs)
    return list(dict.fromkeys(out + RAW))


# ---- tests ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_calls_payloads_bodies_records_and_endpoint(us, name):
    """every binding failure, escaped, duplicate and folded keys, non-list args and non-object kwargs in bodies, kwargs
    beside other keys, callback_url / context / empty / non-ASCII keys: the device answers most of it and agrees with
    CPython on all it answers"""
    c = corpus()
    check_all(us, name, c, min_share=0.9)


def test_every_binding_failure_is_a_type_error(us):
    """each failure CPython raises while binding is ERROR / TypeError, from every source"""
    cases = {"greet": [call("a", "b", "c"), call(), call("a", bogus=1), call("a", name="b")],
             "probe": [call(1, 2, d=3, f=1), call(a=1, b=2, d=3), call(1, 2, 3, c=1, d=1), call(1, 2)],
             "join": [call(sep="-", parts=["a"])], "field_sum": [call([{"x": 1}], "x"), call([{"x": 1}])]}
    for name, calls in cases.items():
        for args, kwargs in calls:
            with pytest.raises(TypeError):
                FNS[name](*args, **kwargs)
            bodies = renderings(args, kwargs)
            # (the third rendering, kwargs as top-level keys, is an HTTP body: as an SDK payload Go ignores those keys)
            assert all(g[:3] == (ERROR, 0, 0x01) for g in us(bodies[:2], name, TQ)), (name, args, kwargs)
            assert all(g[:3] == (ERROR, 0, 0x01) for g in us(bodies, name, TQ, TF_HTTP_BODY)), (name, args, kwargs)
            assert all(g[:3] == (ERROR, 0, 0x01) for g in us(bodies, name, ENDPOINT, TF_HTTP_BODY))
            recs, ids = U.records_of(bodies[:2])
            assert all(g[:3] == (ERROR, 0, 0x01) for g in us(recs, name, TQ, TF_TASK_MSG, ids))


def test_examples_answer(us):
    got = us([sdk(["Ada"], {}), sdk([], {"name": "Ada", "punct": "?"}), b'{"name": "Ada", "greeting": "Hi"}'], "greet", TQ, TF_HTTP_BODY)
    assert [g[3] for g in got] == [b'"Hello, Ada!"', b'"Hello, Ada?"', b'"Hi, Ada!"']
    assert us([sdk(["-", "a", "b"], {})], "join", ENDPOINT, TF_HTTP_BODY)[0][3] == b'"a-b"'
    assert us([sdk([[{"x": 1}, {"x": 2.5}]], {"field": "x"})], "field_sum", TQ)[0][3] == b"3.5"
    assert us([sdk([[{"x": 1}, {"y": 2}]], {"field": "x"})], "field_sum", TQ)[0][:3] == (ERROR, 0, 0x08)   # KeyError
    assert us([sdk([[{"x": 2**62}, {"x": 2**62}]], {"field": "x"})], "field_sum", TQ)[0][0] == UNSUPPORTED


def test_pickle_and_foreign_flags_are_unsupported(us):
    ps = [sdk(["a"], {}), sdk(["a"], {"punct": "?"})]
    for name in NAMES:
        for fl in (0x04, 0x04 | 0x02):
            assert all(g[0] == UNSUPPORTED for g in us(ps, name, TQ, fl))
        for fl in (0, 0x04, 0x08):
            assert all(g[0] == UNSUPPORTED for g in us(ps, name, ENDPOINT, fl))


_key = st.sampled_from(["name", "greeting", "punct", "sep", "parts", "rows", "field", "a", "b", "c", "d", "e", "rest", "args",
                        "kwargs", "context", "callback_url", "", "é", "x"]) | st.text(max_size=4)
_scalar = st.text(max_size=6) | st.integers(min_value=-2**64, max_value=2**64) | st.floats() | st.booleans() | st.none()
_row = st.dictionaries(st.sampled_from(["x", "y", "é", ""]), _scalar, max_size=3)
_val = _scalar | st.lists(_row, max_size=4) | st.lists(st.text(max_size=3), max_size=3) | _row


@settings(max_examples=400, deadline=None, suppress_health_check=list(HealthCheck))
@given(args=st.lists(_val, max_size=5), kwargs=st.dictionaries(_key, _val, max_size=4), ascii_=st.booleans())
def test_hypothesis_calls(us, args, kwargs, ascii_):
    bodies = []
    for b in renderings(args, kwargs):
        try:
            bodies.append(json.dumps(json.loads(b), ensure_ascii=ascii_).encode("utf-8", "surrogatepass"))
        except ValueError:
            pass
    for name in NAMES:
        check_all(us, name, bodies)


@pytest.mark.parametrize("name", NAMES)
def test_single_byte_mutations(us, name):
    """30 k payloads with one byte replaced, deleted or inserted, over the four handlers"""
    base = [b for b in corpus() if len(b) >= 4]
    rng = np.random.default_rng(71 + NAMES.index(name))
    alphabet = list(b'{}[],:" 01e.-nulltrackwgsAv\\\x7fxdyfi') + [0xC3, 0xA9, 0xFF, 0x1F]
    bodies = []
    while len(bodies) < 30000 // len(NAMES):
        m = bytearray(base[int(rng.integers(0, len(base)))])
        pos = int(rng.integers(0, len(m)))
        op = int(rng.integers(0, 3))
        ch = int(rng.choice(alphabet))
        if op == 0: m[pos] = ch
        elif op == 1: del m[pos]
        else: m[pos:pos] = bytes([ch])
        bodies.append(bytes(m))
    check_tq(us, name, bodies)
    check_tq(us, name, bodies, http=True)
    check_ep(us, name, bodies)


def test_two_passes_must_agree(us):
    """a string result binds the call again in phase B: it must see the values phase A saw"""
    for name in NAMES:
        for fl in (0, TF_HTTP_BODY):
            assert all(g[0] != 255 for g in us(corpus(), name, TQ, fl))


# ---- compile-time checks of B9H_SIGNATURE ---------------------------------------------------------------------------------
BAD_SIGNATURES = {
    "at most 8": ", ".join('B9H_POS_OR_KW_OPT("p%d")' % i for i in range(9)),
    "ASCII identifiers": 'B9H_POS_OR_KW("1x")',
    "identifiers ": 'B9H_POS_OR_KW("na-me")',
    "duplicate": 'B9H_POS_OR_KW("x"), B9H_KW_ONLY("x")',
    "context": 'B9H_POS_OR_KW("x"), B9H_KW_ONLY_OPT("context")',
    "positional-only, positional-or-keyword": 'B9H_KW_ONLY("x"), B9H_POS_OR_KW("y")',
    "positional defaults last": 'B9H_POS_OR_KW_OPT("x"), B9H_POS_OR_KW("y")',
    "*args": 'B9H_VAR_POS("x"), B9H_VAR_POS("y")',
}
TEMPLATE = """#include "b9gpu_handler.cuh"
struct S { B9H_SIGNATURE(%s);
    template <class Out> __device__ static int call(const b9h::Call&, Out&) { return 0; } };
static_assert(b9h::has_signature<S>::value, "");
"""
GPP_PRELUDE = "#include <stdint.h>\n#include <string.h>\n#define __device__\n#define __host__\n#define __forceinline__ inline\n" \
              "#define __noinline__\n#define __restrict__\n#define __constant__ static const\n" \
              "static inline float __uint_as_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }\n" \
              "static inline uint32_t __float_as_uint(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }\n" \
              "static inline float __fadd_rn(float a, float b) { return a + b; }\n"


def _compile(tmp_path, body, nvcc):
    src = tmp_path / ("s.cu" if nvcc else "s.cpp")
    src.write_text(body if nvcc else GPP_PRELUDE + body)
    inc = "-I" + os.path.join(ROOT, "include")
    if nvcc:
        from beta9_b200 import build as B
        cmd = [B.NVCC, "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-cubin", inc, "-o", str(tmp_path / "s.cubin"), str(src)]
    else:
        cmd = [U.GXX, "-std=c++17", "-fsyntax-only", "-w", inc, str(src)]
    return subprocess.run(cmd, capture_output=True, text=True)


@pytest.mark.parametrize("what", list(BAD_SIGNATURES))
def test_bad_signatures_do_not_compile_with_gxx(tmp_path, what):
    if shutil.which(U.GXX) is None:
        pytest.skip("no host C++ compiler")
    ok = _compile(tmp_path, TEMPLATE % 'B9H_POS_ONLY("a"), B9H_POS_OR_KW_OPT("b"), B9H_VAR_POS("c"), B9H_KW_ONLY("d")', False)
    assert ok.returncode == 0, ok.stderr[-2000:]
    r = _compile(tmp_path, TEMPLATE % BAD_SIGNATURES[what], False)
    assert r.returncode != 0 and re.search(re.escape(what.strip()), r.stderr), r.stderr[-2000:]


def test_bad_signatures_do_not_compile_with_nvcc(tmp_path):
    from beta9_b200 import build as B
    if not os.path.exists(B.NVCC):
        pytest.skip("no nvcc")
    ok = _compile(tmp_path, TEMPLATE % 'B9H_POS_OR_KW("a"), B9H_KW_ONLY_OPT("b")', True)
    assert ok.returncode == 0, ok.stderr[-2000:]
    for what in ("context", "at most 8"):
        r = _compile(tmp_path, TEMPLATE % BAD_SIGNATURES[what], True)
        assert r.returncode != 0 and what in r.stderr, r.stderr[-2000:]


def test_example_cubin_exports_the_signature_handlers():
    from beta9_b200 import build as B
    if not os.path.exists(B.NVCC):
        pytest.skip("no nvcc")
    out = B.build_examples()
    cuobjdump = shutil.which("cuobjdump") or os.path.join(os.path.dirname(B.NVCC), "cuobjdump")
    syms = subprocess.run([cuobjdump, "-symbols", out], capture_output=True, text=True).stdout
    v = B.handler_abi_version()
    for name in ("greet", "join", "field_sum"):
        for kind in ("tq", "ep"):
            assert f"b9h_v{v}_{kind}_{name}" in syms, (name, kind)
