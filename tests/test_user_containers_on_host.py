"""User handlers that return lists and dicts, on a CPU: the sinks' container calls (list_begin / list_end, dict_begin /
dict_end, value) in include/b9gpu_handler.cuh, compiled for the host by tests/host_shim/user_containers_shim.cpp with the
container script handler (tests/handlers/containers.cuh) and the examples tokens, grid, describe and pick
(examples/handlers/handlers.cuh).

cscript's twin (tests/handlers/container_twins.py) states the rules and predicts the Python value a script builds; the
runner's own loops render it, so the device's bytes are checked against CPython's json. The examples run against their
twins in examples/handlers/handlers.py over the user-handler corpora of tests/test_user_handler_on_host.py. No writing
pass may touch a byte past its record's reservation. The corpora are functions of this module so that
tests/test_gpu_user_containers.py runs the same ones on the device."""
import ctypes as C
import json
import os

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from oracle.pyoracle import endpoint as EP
from tests import test_handler_contract_on_host as H
from tests import test_user_handler_on_host as U
from tests import test_user_signature_on_host as S
from tests.handlers import container_twins as T

HERE, ROOT = U.HERE, U.ROOT
SRC = os.path.join(HERE, "host_shim", "user_containers_shim.cpp")
SO = os.path.join(HERE, "host_shim", "libusercontainersshim.so")
NAMES = ["tokens", "grid", "describe", "pick", "cscript"]
EXAMPLES = NAMES[:4]
COMPLETE, ERROR, REJECTED, UNSUPPORTED = U.COMPLETE, U.ERROR, U.REJECTED, U.UNSUPPORTED
TF_HTTP_BODY, TF_TASK_MSG, TQ, ENDPOINT = U.TF_HTTP_BODY, U.TF_TASK_MSG, U.TQ, U.ENDPOINT
op = H.op


@pytest.fixture(scope="module")
def uc():
    lib = U._shim(SRC, SO, ["-I" + os.path.join(ROOT, "include")])
    u64p, u8p, i64p = (np.ctypeslib.ndpointer(t, flags="C") for t in (np.uint64, np.uint8, np.int64))
    lib.b9_uc_batch.argtypes = [C.c_char_p, u64p, u8p, u8p, C.c_uint32, C.c_int, C.c_int, u8p, u8p, i64p, u8p, C.c_void_p, u64p]
    lib.b9_uc_batch.restype = C.c_uint64

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
        total = lib.b9_uc_batch(blob, off, fl, idb, n, h, rendering, status, has, val, guard, None, out_off)
        out = np.zeros(total + 1, np.uint8)
        lib.b9_uc_batch(blob, off, fl, idb, n, h, rendering, status, has, val, guard, out.ctypes.data, out_off)
        assert guard.all(), [payloads[i] for i in np.flatnonzero(guard == 0)[:5]]
        raw = out.tobytes()
        return [(int(status[i]), int(has[i]), int(val[i]), raw[int(out_off[i]):int(out_off[i + 1])] if has[i] else b"")
                for i in range(n)]
    return batch


# ---- when may the examples decline? -------------------------------------------------------------------------------------
def _repeated_keys(keys):
    """pick's declared decline: two equal str keys (the built dict would hold two equal keys)"""
    ks = [k for k in keys if type(k) is str]
    return len(set(ks)) != len(ks)


def may_decline(name, payload, args, kwargs=None):
    """the example handlers' documented declines: test_user_handler_on_host's (long literals, deep nesting), a
    signature's (kwargs objects Go merges), value()
    where identity declines (nesting past 16 non-empty containers, a dict of more than 64 members), pick's repeated keys"""
    if U._long_literal(payload) or (name == "pick" and S._kwargs_merged(payload)):
        return True
    if name in ("describe", "pick") and args:
        vals = list(args) + list((kwargs or {}).values())
        if any(T.identity_declines(v) for v in vals):
            return True
        if name == "pick" and _repeated_keys(args[1:]):
            return True
    return False


@pytest.fixture(scope="module", autouse=True)
def _examples_rules():
    """test_user_handler_on_host's comparisons, with the exception class of any call (pick takes *keys) and the
    declines of the container examples"""
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(U, "may_decline", lambda name, payload, args: may_decline(name, payload, args))
        mp.setattr(U, "exc_bit", S.exc_bit)
        yield


# ---- the examples -------------------------------------------------------------------------------------------------------
def example_calls():
    """calls that reach each example's branches: words and lines with every space, every kind of argument, pick's keys"""
    d = {"a": 1, "b": [1, "x", None], "é": {"z": 2.5, "y": True}, "": "", "\U0001F600": -0.0, "c": {"b": 1, "a": 2}}
    strs = ["", " ", "a", "hello world", "  a  b  ", U.SPACES, "x" + U.SPACES + "y", "a\nb", "a\n\nb\n", "\n", " \n ",
            "l1 w1 w2\nl2\r\nl3\x0bx", "café \U0001F600 \"q\" \\", "\x00\x1f\x7f", "ab cd ", "　x　"]
    calls = [((s,), {}) for s in strs]
    calls += [((v,), {}) for v in [None, True, False, 0, -1, 2**53, 1.5, -0.0, 1e21, 1e-7, [], {}, [1, [2, [3]]], d,
                                   {"b": 1, "a": 2, "A": 3}, [{}], [[]], "x" * 300]]
    calls += [((d,) + ks, {}) for ks in [(), ("a",), ("a", "b"), ("é", "\U0001F600", ""), ("c",), ("zz",), ("a", "zz"),
                                         ("a", 1), ("a", None), ("a", [1]), ("a", {"a": 1}), ("a", "a"), ("b", "a", "b")]]
    calls += [((v, "a"), {}) for v in ([1], "a", None, 3)] + [(([1],), {}), ((), {}), (("a", "b"), {}), ((d,), {"keys": ["a"]}),
                                                              ((), {"d": d})]
    return calls


def example_payloads():
    out = []
    for args, kwargs in example_calls():
        out += [json.dumps({"args": list(args), "kwargs": kwargs}).encode(),
                json.dumps({"args": list(args), "kwargs": kwargs}, ensure_ascii=False).encode()]
    out += [b'{"args": [{"a": 1, "a": 2}, "a"]}', b'{"args": [{"\\u0061": 1, "a": [2]}, "\\u0061", "b"]}',
            b'{"args": [{"a": 1}, "a", "\\u0061"]}', b'{"args": [{"x": 12345678901234567890123}, "x"]}',
            b'{"args": [{"b": 1, "a": 2, "b": 3}]}', b'{"args": ["\\ud800 \\udc00x"]}', b'{"args": ["a\xffb c"]}']
    return list(dict.fromkeys(out))


def check_example(run, name, payloads, min_share=0.0):
    """SDK payloads, HTTP bodies, TaskMessage records and endpoint requests through test_user_handler_on_host's checks"""
    a = U.check_tq(run, name, payloads)
    b = U.check_tq(run, name, payloads, http=True)
    c = U.check_ep(run, name, payloads)
    recs, ids = U.records_of(payloads)
    d = U.check_records(run, name, recs, ids)
    assert min(a, b, c) >= min_share * len(payloads) and d >= min_share * len(recs), (name, a, b, c, d)


@pytest.mark.parametrize("name", EXAMPLES)
def test_examples_over_their_calls(uc, name):
    check_example(uc, name, example_payloads(), 0.5)


@pytest.mark.parametrize("name", EXAMPLES)
def test_examples_over_the_user_handler_corpus(uc, name):
    c = U.corpus()
    check_example(uc, name, c, 0.8)


@pytest.mark.parametrize("name", EXAMPLES)
def test_examples_single_byte_mutations(uc, name):
    """30 k payloads with one byte replaced, deleted or inserted, over the four examples"""
    base = [b for b in U.corpus() + example_payloads() if len(b) >= 4]
    rng = np.random.default_rng(91 + EXAMPLES.index(name))
    alphabet = list(b'{}[],:" 01e.-nulltrackwgsAv\\\x7f\t\nab') + [0xC3, 0xA9, 0xFF, 0x1F, 0xE3, 0x80]
    bodies = []
    while len(bodies) < 30000 // len(EXAMPLES):
        m = bytearray(base[int(rng.integers(0, len(base)))])
        pos = int(rng.integers(0, len(m)))
        k = int(rng.integers(0, 3))
        ch = int(rng.choice(alphabet))
        if k == 0: m[pos] = ch
        elif k == 1: del m[pos]
        else: m[pos:pos] = bytes([ch])
        bodies.append(bytes(m))
    U.check_tq(uc, name, bodies)
    U.check_ep(uc, name, bodies)


@settings(max_examples=300, deadline=None, suppress_health_check=list(HealthCheck))
@given(v=U._arg, keys=st.lists(st.text(max_size=2) | st.integers(-2, 2) | st.none(), max_size=3), ascii_=st.booleans())
def test_hypothesis_values(uc, v, keys, ascii_):
    bodies = []
    for args in ([v], [v] + keys, [{"k": v, "": [v]}] + keys):
        try:
            bodies.append(json.dumps({"args": args, "kwargs": {}}, ensure_ascii=ascii_).encode("utf-8", "surrogatepass"))
        except ValueError:
            pass
    for name in EXAMPLES:
        check_example(uc, name, bodies)


def test_describe_value_is_identitys_record(uc):
    """describe's "value" member is byte for byte the record the built-in identity host build writes for the same task
    (truthy arguments: identity writes no bytes for a falsy one)"""
    hp = U._shim(os.path.join(HERE, "host_shim", "host_parse.cpp"), os.path.join(HERE, "host_shim", "libhostparse_uc.so"))
    hp.b9_host_run.argtypes = [C.c_char_p, C.c_uint32, C.c_int, C.c_int, C.POINTER(C.c_uint8), C.POINTER(C.c_uint8), C.c_void_p, C.c_uint32]
    hp.b9_host_run.restype = C.c_long
    payloads = U.corpus() + example_payloads()
    checked = 0
    for http in (0, 1):
        got = uc(payloads, "describe", TQ, TF_HTTP_BODY if http else 0)
        for p, (st_, has, _, data) in zip(payloads, got):
            s_, h_ = C.c_uint8(), C.c_uint8()
            buf = (C.c_uint8 * (len(p) * 12 + 64))()
            n = hp.b9_host_run(p, len(p), http, 0, C.byref(s_), C.byref(h_), buf, len(buf))
            if st_ != COMPLETE or s_.value != COMPLETE or not h_.value:
                continue
            name = json.loads(data)["type"]
            prefix = b'{"type": ' + json.dumps(name).encode() + b', "value": '
            assert data == prefix + bytes(buf[:n]) + b"}", (p, data, bytes(buf[:n]))
            checked += 1
    assert checked > len(payloads) // 2


def test_examples_answer(uc):
    got = uc([U.sdk("a b　c"), U.sdk("x\ny z\n"), U.sdk("")], "tokens", TQ)
    assert [g[3] for g in got] == [b'["a", "b", "c"]', b'["x", "y", "z"]', b""]
    assert uc([U.sdk("x\ny z\n")], "grid", ENDPOINT, TF_HTTP_BODY)[0][3] == b'[["x"],["y","z"],[]]'
    assert uc([U.sdk([1, {"b": 2, "a": 1}])], "describe", TQ)[0][3] == b'{"type": "list", "value": [1, {"a": 1, "b": 2}]}'
    assert uc([U.sdk(None)], "describe", ENDPOINT, TF_HTTP_BODY)[0][3] == b'{"type":"NoneType","value":null}'
    d = {"a": 1, "é": [2]}
    assert uc([U.sdk(d, "é", "a")], "pick", ENDPOINT, TF_HTTP_BODY)[0][3] == '{"é":[2],"a":1}'.encode()
    assert uc([U.sdk(d, "é", "a")], "pick", TQ)[0][3] == b'{"\\u00e9": [2], "a": 1}'
    assert uc([U.sdk(d)], "pick", TQ)[0][:2] == (COMPLETE, 0)                  # {} is falsy
    assert uc([U.sdk(d, "zz")], "pick", TQ)[0][:3] == (ERROR, 0, 0x08)
    assert uc([U.sdk(d, ["a"])], "pick", TQ)[0][:3] == (ERROR, 0, 0x01)
    assert uc([U.sdk([1], "a")], "pick", TQ)[0][:3] == (ERROR, 0, 0x01)
    assert uc([U.sdk(d, "a", "a")], "pick", TQ)[0][0] == UNSUPPORTED
    assert uc([b'{"args": [{"a": 1}, "a", "\\u0061"]}'], "pick", TQ)[0][0] == UNSUPPORTED


# ---- cscript ----------------------------------------------------------------------------------------------------------------
LB, LE, DB, DE = op(T.LIST_BEGIN), op(T.LIST_END), op(T.DICT_BEGIN), op(T.DICT_END)
SB, SE = op(T.STR_BEGIN), op(T.STR_END)


def key(s):
    return [SB] + [op(T.CP, ord(c)) for c in s] + [SE]


# the values cscript passes through with value(): every kind, one of each edge
REST = [0, 1, -0.0, 2.5, 1e21, "", "a\"\\\né\U0001F600", None, True, False, [], {}, [1, [2, [3, {"b": 1, "a": [None]}]]],
        {"b": 1, "a": 2, "é": "x"}, 2**53 + 2, -7]
OPS = [op(T.NONE), op(T.BOOL, 1), op(T.BOOL, 0), op(T.INT, 0), op(T.INT, -5), op(T.INT, H.T.INT64_MIN), op(T.REAL, H.bits(1.5)),
       op(T.REAL, 0x7FF8000000000000), op(T.REAL, 0xFFF0000000000000), op(T.REAL, 0x8000000000000000), SB, op(T.CP, 0x41),
       op(T.CP, 0xE9), op(T.CP, 0xD800), SE, op(T.RETURN, 0), op(T.RETURN, 8), op(T.RETURN, -1), op(T.CP_WRITE, 0x41),
       op(T.CP_COUNT, 0x42), LB, LE, DB, DE] + [op(T.VALUE_OF, k) for k in (0, 1, 5, 6, 7, 10, 12, 13)]


def pair_scripts():
    """every op and every ordered pair of ops: alone, in a list, as a dict's value and after a dict's key"""
    out = []
    for a in OPS:
        for seq in [[a]] + [[a, b] for b in OPS]:
            out += [seq, [LB] + seq + [LE], [DB] + key("k") + seq + [DE], [DB] + seq + [DE]]
    return out


def random_scripts(n, seed):
    """n random scripts of up to 24 ops, mostly well nested containers of strings, scalars and values, now and then a
    broken rule"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        ops, stack = [], []
        for _ in range(int(rng.integers(0, 24))):
            r = rng.random()
            if r < 0.15 and len(stack) < 18:
                d = rng.random() < 0.5
                ops.append(DB if d else LB)
                stack.append("d" if d else "l")
            elif r < 0.3 and stack:
                ops.append(DE if stack.pop() == "d" else LE)
            elif stack and stack[-1] == "d" and rng.random() < 0.8:
                ops += key(rng.choice(["a", "b", "é", "", "a\"", "\U0001F600"]))
                ops += [op(T.VALUE_OF, int(rng.integers(0, len(REST))))] if rng.random() < 0.5 else key("v")
            elif r < 0.5:
                ops.append(op(T.VALUE_OF, int(rng.integers(0, len(REST)))))
            elif r < 0.65:
                ops += [SB] + [op(T.CP, H._cp_pool(rng)) for _ in range(int(rng.integers(0, 4)))] + [SE]
            else:
                ops.append(OPS[int(rng.integers(0, len(OPS)))])
        if rng.random() < 0.8:
            ops += [DE if s == "d" else LE for s in reversed(stack)]
        out.append(ops)
    return out


def script_outcome(rendering):
    def outcome(args, kwargs):
        kind, x = T.expect(args[0], args[1:], rendering)
        return kind, x if kind == T.ERROR else 0
    return outcome


def check_scripts(run, scripts, rest=REST):
    """every script from every source against expect and the runner's rendering"""
    payloads = [json.dumps({"args": [s] + list(rest), "kwargs": {}}).encode() for s in scripts]
    for source, rendering, flags, ps, ids in H.sources_of(payloads):
        want = H.expected(T.twin(rendering), source, rendering, ps, ids, script_outcome(rendering))
        got = run(ps, "cscript", rendering, flags, ids)
        for s, g, w in zip(scripts, got, want):
            assert H.same(g, w), (source, s, g, w)


def test_every_op_and_pair_of_ops(uc):
    check_scripts(uc, pair_scripts())


def test_random_scripts(uc):
    check_scripts(uc, random_scripts(4000, 5))


def run_one(uc, ops, rendering, rest=REST):
    flags = TF_HTTP_BODY if rendering == ENDPOINT else 0
    return uc([json.dumps({"args": [ops] + list(rest), "kwargs": {}}).encode()], "cscript", rendering, flags)[0]


BROKEN = {
    "a close with no open container": [[LE], [DE], [LB, LE, LE], [op(T.INT, 1), LE]],
    "a close of the wrong kind": [[LB, DE], [DB, LE], [LB, DB, LE, DE]],
    "a result left open": [[LB], [DB], [LB, DB] + key("a") + [op(T.INT, 1), DE], [LB, SB]],
    "dict_end after a key with no value": [[DB] + key("a") + [DE], [DB] + key("a") + [op(T.INT, 1)] + key("b") + [DE]],
    "a non-string key": [[DB, op(T.INT, 1), op(T.INT, 2), DE], [DB, op(T.NONE), DE], [DB, LB, LE, op(T.INT, 1), DE],
                         [DB, op(T.VALUE_OF, 5), op(T.INT, 1), DE], [DB, op(T.VALUE_OF, 6), op(T.INT, 1), DE]],
    "a container call while a string is open": [[SB, LB, LE, SE], [LB, SB, LE], [DB, SB, DE], [LB, SB, op(T.VALUE_OF, 5), SE, LE],
                                                [DB, SB, op(T.CP, 0x61), op(T.INT, 1), SE, DE]],
    "a second top-level value": [[LB, LE, LB, LE], [op(T.INT, 1), LB, LE], [DB, DE, op(T.VALUE_OF, 1)],
                                 [op(T.VALUE_OF, 1), op(T.VALUE_OF, 1)], [SB, SE, DB, DE]],
    "a 17th open container": [[LB] * 17 + [LE] * 17, [DB] + sum([key("a") + [DB] for _ in range(16)], []) + [DE] * 17],
    "65 members": [[DB] + sum([key("k%d" % i) + [op(T.INT, i)] for i in range(65)], []) + [DE]],
    "two equal keys": [[DB] + key("a") + [op(T.INT, 1)] + key("a") + [op(T.INT, 2), DE],
                       [LB, DB] + key("é") + [LB, LE] + key("x") + [op(T.NONE)] + key("é") + [op(T.INT, 2), DE, LE]],
    "a writing pass of another length": [[LB, SB, op(T.CP, 0x41), op(T.CP_WRITE, 0x42), SE, LE],
                                         [DB, SB, op(T.CP_COUNT, 0x41), SE, op(T.INT, 1), DE]],
}


def test_broken_rules_are_unsupported(uc):
    for rule, scripts in BROKEN.items():
        for ops in scripts:
            for rendering in (TQ, ENDPOINT):
                assert T.expect(ops, REST, rendering) == (T.UNSUPPORTED, None), (rule, ops)
                assert run_one(uc, ops, rendering) == (UNSUPPORTED, 0, 0, b""), (rule, ops, rendering)


def test_depth_and_member_limits(uc):
    """16 open containers and 64 members are written; 17 and 65 are UNSUPPORTED (BROKEN)"""
    deep = [LB] * 16 + [op(T.INT, 1)] + [LE] * 16
    assert run_one(uc, deep, TQ)[3] == b"[" * 16 + b"1" + b"]" * 16
    assert run_one(uc, [DB] + key("a") + [LB] * 15 + [LE] * 15 + [DE], ENDPOINT)[3] == b'{"a":' + b"[" * 15 + b"]" * 15 + b"}"
    wide = [DB] + sum([key("k%d" % i) + [op(T.INT, i)] for i in range(64)], []) + [DE]
    assert json.loads(run_one(uc, wide, TQ)[3]) == {"k%d" % i: i for i in range(64)}
    # value() of an argument nested 16 deep inside 16 built containers: identity's limit is its own
    v = [[[[[[[[[[[[[[[[1]]]]]]]]]]]]]]]]
    got = run_one(uc, [LB] * 16 + [op(T.VALUE_OF, 0)] + [LE] * 16, TQ, [v])
    assert got[3] == b"[" * 16 + json.dumps(v).encode() + b"]" * 16
    assert run_one(uc, [op(T.VALUE_OF, 0)], TQ, [[v]]) == (UNSUPPORTED, 0, 0, b"")
    assert run_one(uc, [op(T.VALUE_OF, 0)], TQ, [{"k%d" % i: i for i in range(65)}]) == (UNSUPPORTED, 0, 0, b"")


def test_non_finite_floats_inside_containers(uc):
    for b, tq in ((0x7FF8000000000000, b"NaN"), (0xFFF8000000000001, b"NaN"), (0x7FF0000000000000, b"Infinity"),
                  (0xFFF0000000000000, b"-Infinity")):
        for ops, want in (([LB, op(T.REAL, b), LE], b"[%s]" % tq), ([DB] + key("x") + [LB, op(T.REAL, b), LE, DE], b'{"x": [%s]}' % tq)):
            assert run_one(uc, ops, TQ) == (COMPLETE, 1, 0, want)
            assert run_one(uc, ops, ENDPOINT) == (UNSUPPORTED, 0, 0, b"")


def test_falsy_containers_and_values(uc):
    """a top-level [] or {} is COMPLETE without bytes in the task queue, a body in the endpoint; value(a) is falsy exactly
    where identity drops a"""
    for ops, ep in (([LB, LE], b"[]"), ([DB, DE], b"{}")):
        assert run_one(uc, ops, TQ) == (COMPLETE, 0, 0, b"")
        assert run_one(uc, ops, ENDPOINT) == (COMPLETE, 1, 0, ep)
    for k, v in enumerate(REST):
        assert run_one(uc, [op(T.VALUE_OF, k)], TQ)[1] == (1 if v else 0), v
        assert run_one(uc, [op(T.VALUE_OF, k)], ENDPOINT)[1] == 1
    assert run_one(uc, [LB, LB, LE, LE], TQ) == (COMPLETE, 1, 0, b"[[]]")


def test_value_writes_identitys_bytes(uc):
    """value(a) at the top level and inside a list is the built-in identity host build's record for a; in the endpoint
    rendering, the runner's identity response"""
    hp = U._shim(os.path.join(HERE, "host_shim", "host_parse.cpp"), os.path.join(HERE, "host_shim", "libhostparse_uc.so"))
    hp.b9_host_run.argtypes = [C.c_char_p, C.c_uint32, C.c_int, C.c_int, C.POINTER(C.c_uint8), C.POINTER(C.c_uint8), C.c_void_p, C.c_uint32]
    hp.b9_host_run.restype = C.c_long
    for v in REST + ["x" * 300, [0.1, -0.0, 1e-7, 2**60], {"\u2028": "<&>", "b": [{}], "a": None}]:
        p = json.dumps({"args": [v], "kwargs": {}}).encode()
        s_, h_ = C.c_uint8(), C.c_uint8()
        buf = (C.c_uint8 * 4096)()
        n = hp.b9_host_run(p, len(p), 0, 0, C.byref(s_), C.byref(h_), buf, len(buf))
        ident = bytes(buf[:n]) if h_.value else b""
        assert run_one(uc, [op(T.VALUE_OF, 0)], TQ, [v])[3] == ident, v
        if ident:
            assert run_one(uc, [LB, op(T.VALUE_OF, 0), op(T.VALUE_OF, 0), LE], TQ, [v])[3] == b"[%s, %s]" % (ident, ident)
        ep = run_one(uc, [op(T.VALUE_OF, 0)], ENDPOINT, [v])[3]
        assert ep == EP.run_endpoint_request(p, lambda x, /: x)[1], v                  # (the runner's identity)
