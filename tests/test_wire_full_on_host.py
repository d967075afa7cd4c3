"""b9_wire_encode_full's Args and Kwargs on a CPU: the payload parser, go_transcode, the ordered Go walk (go_value_json)
and the HTTP kwargs rule, compiled for the host by tests/host_shim/wire_full_shim.cpp, against the oracle's Go encoder
(gojson.go_marshal of go_unmarshal_task_payload / serialize_http_payload).

Everywhere: the device's bytes are the oracle's; a decline has one of the documented reasons (merged struct kwargs, a
literal of more than 19 significant digits, nesting deeper than 16, an object of more than 64 members); and wherever
go_transcode answers a value, the walk over the same span writes the same bytes."""
import ctypes as C
import json
import math
import os
import random
import subprocess

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from oracle.pyoracle.gojson import GoJSONError, go_fold_equal, go_format_float64, go_marshal, go_unmarshal_task_payload
from oracle.pyoracle.httpserialize import InvalidRequestPayload, serialize_http_payload
from tests.f64_corpus import _literals, _nest, _sig_digits, _wide, sum_edge_payloads, value_edge_payloads

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_shim", "wire_full_shim.cpp")
SO = os.path.join(HERE, "host_shim", "libwirefull.so")
GXX = os.environ.get("CXX", "g++")
OK, REJECTED, UNSUPPORTED = 0, 3, 4


@pytest.fixture(scope="module")
def wf():
    csrc = os.path.join(os.path.dirname(HERE), "beta9_b200", "csrc")
    deps = [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".h"))]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max([os.path.getmtime(SRC)] + [os.path.getmtime(d) for d in deps]):
        r = subprocess.run([GXX, "-O2", "-std=c++17", "-shared", "-fPIC", "-o", SO, SRC], capture_output=True, text=True)
        if r.returncode:
            pytest.skip("no host C++ compiler for the shim: " + r.stderr[-300:])
    lib = C.CDLL(SO)
    u64p, u8p = np.ctypeslib.ndpointer(np.uint64, flags="C"), np.ctypeslib.ndpointer(np.uint8, flags="C")
    lib.b9_wf_batch.argtypes = [C.c_char_p, u64p, C.c_uint32, C.c_int, u8p, u8p, u8p, u8p, C.c_void_p, u64p]
    lib.b9_wf_batch.restype = C.c_uint64
    lib.b9_wf_walk.argtypes = [C.c_char_p, C.c_uint32, C.c_int, C.c_char_p, C.c_uint32]
    lib.b9_wf_walk.restype = C.c_long
    lib.b9_wf_transcode.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32]
    lib.b9_wf_transcode.restype = C.c_long

    class WF:
        @staticmethod
        def batch(payloads, http: bool):
            """[(status, kw_merged, args bytes, kwargs bytes, walk agrees, (args mode, kwargs mode))] per payload"""
            n = len(payloads)
            off = np.zeros(n + 1, np.uint64)
            np.cumsum([len(p) for p in payloads], out=off[1:])
            blob = b"".join(payloads)
            status, merged, agree = np.zeros(n, np.uint8), np.zeros(n, np.uint8), np.zeros(n, np.uint8)
            mode = np.zeros(2 * n, np.uint8)
            out_off = np.zeros(n + 1, np.uint64)
            total = lib.b9_wf_batch(blob, off, n, int(http), status, merged, mode, agree, None, out_off)
            out = np.zeros(total + 1, np.uint8)
            lib.b9_wf_batch(blob, off, n, int(http), status, merged, mode, agree, out.ctypes.data, out_off)
            raw = out.tobytes()
            res = []
            for i in range(n):
                a = k = None
                if status[i] == OK:
                    a, k = raw[int(out_off[i]):int(out_off[i + 1])].split(b"\x00")
                res.append((int(status[i]), int(merged[i]), a, k, int(agree[i]), (int(mode[2 * i]), int(mode[2 * i + 1]))))
            return res

        @staticmethod
        def walk(tok: bytes, drop_args: bool = False):
            buf = C.create_string_buffer(8 * len(tok) + 64)
            n = lib.b9_wf_walk(tok, len(tok), int(drop_args), buf, len(buf))
            assert n != -2
            return None if n < 0 else buf.raw[:n]

        @staticmethod
        def transcode(tok: bytes):
            buf = C.create_string_buffer(8 * len(tok) + 64)
            n = lib.b9_wf_transcode(tok, len(tok), buf, len(buf))
            return None if n < 0 else buf.raw[:n]
    return WF


def go_record_values(b: bytes, http: bool):
    """(Args, Kwargs) as TaskMessage.Encode writes them, or None where Go refuses the payload"""
    try:
        args, kwargs = serialize_http_payload(b) if http else go_unmarshal_task_payload(b)
    except (GoJSONError, InvalidRequestPayload):
        return None
    return go_marshal(args if args is not None else []).encode(), go_marshal(kwargs).encode()


def _kw_merged(b: bytes) -> bool:
    """an SDK payload with more than one top-level object under a key that folds to "kwargs": Go merges the maps"""
    try:
        top = json.loads(b.decode("utf-8", "replace"), object_pairs_hook=lambda ps: ("obj", ps))
    except ValueError:
        return False
    return isinstance(top, tuple) and sum(1 for k, v in top[1] if go_fold_equal(k, "kwargs") and isinstance(v, tuple)) > 1


def decline_reasons(b: bytes, http: bool, kw_merged: bool = None):
    """The documented reasons the device may have for declining payload b (kw_merged: the parser's flag, if known)"""
    reasons = set()
    if not http and (kw_merged if kw_merged is not None else _kw_merged(b)):
        reasons.add("kw_merged")

    def num(s):
        if _sig_digits(s) > 19:
            reasons.add("digits")
        return 0

    def pairs(ps):
        if len(ps) > 64:
            reasons.add("members")
        return ("obj", [v for _, v in ps])
    doc = json.loads(b.decode("utf-8", "replace"), parse_int=num, parse_float=num, object_pairs_hook=pairs)

    def depth(v):
        kids = v[1] if isinstance(v, tuple) else v if isinstance(v, list) else None
        return 0 if not kids else 1 + max(depth(x) for x in kids)
    if depth(doc) > 16:                                   # (the payload's own object is one level above args / kwargs)
        reasons.add("depth")
    return reasons


def _raw_depth(b: bytes) -> int:
    """deepest bracket nesting of b outside string tokens"""
    d = best = 0
    in_str = esc = False
    for c in b:
        if in_str:
            esc, in_str = (False, True) if esc else (c == 0x5C, c != 0x22)
        elif c == 0x22:
            in_str = True
        elif c in b"[{":
            d += 1
            best = max(best, d)
        elif c in b"]}":
            d -= 1
    return best


def check(wf, payloads, http: bool, min_answered: float = 0.5):
    got = wf.batch(payloads, http)
    answered = declined = 0
    for b, (st_, merged, a, k, agree, modes) in zip(payloads, got):
        want = go_record_values(b, http)
        assert agree != 0, b                              # go_transcode answered and the walk wrote other bytes
        if agree == 2:                                    # the walk declined what go_transcode answered: one of its limits
            assert decline_reasons(b, http, merged) & {"depth", "members"}, b
        if st_ == UNSUPPORTED and want is None:           # nesting deeper than the parser's stack: never decided
            assert _raw_depth(b) > 64, b
            declined += 1
            continue
        if st_ == UNSUPPORTED:
            assert decline_reasons(b, http, merged), b
            declined += 1
            continue
        if want is None:
            assert st_ == REJECTED, (b, st_)
            continue
        assert st_ == OK and (a, k) == want, (b, a, k, want)
        answered += 1
    assert answered >= min_answered * (answered + declined), (answered, declined)
    return answered, declined


# ---------------------------------------------------------------------------------------------- corpora
@pytest.mark.parametrize("http", [False, True], ids=["sdk_payload", "http_body"])
def test_fuzz_corpus(wf, http):
    from tests.test_device_parser_on_host import _payloads
    answered, _ = check(wf, _payloads(), http)
    assert answered > 300


def test_every_f64_literal(wf):
    """the 1.05 M literals of the float64 corpus as `{"args": [lit]}`: Go's float64 text of ParseFloat's value"""
    lits = _literals()
    assert len(lits) >= 1_000_000
    payloads = [b'{"args": [' + s.encode() + b"]}" for s in lits]
    got = wf.batch(payloads, False)
    declined = 0
    for lit, (st_, _, a, k, agree, _) in zip(lits, got):
        x = float(lit)
        if math.isinf(x):
            assert st_ == REJECTED, lit
            continue
        if st_ == UNSUPPORTED:
            assert _sig_digits(lit) > 19, lit
            declined += 1
            continue
        assert st_ == OK and a == ("[" + go_format_float64(x) + "]").encode() and k == b"null", (lit, a)
        assert agree == 1, lit
    assert declined <= sum(1 for s in lits if _sig_digits(s) > 19) and declined < len(lits) // 5   # (the corpus seeks out rounding midpoints)


def test_f64_edge_payloads(wf):
    payloads = [p for p, _ in sum_edge_payloads()] + [p for p, _ in value_edge_payloads()]
    check(wf, payloads, False)
    check(wf, payloads, True)


def test_reference_serialize_bodies(wf):
    """pkg/task/serialize_test.go's 15 bodies (the query strings are the host's to merge)"""
    from tests.test_oracle_reference_answers import SERIALIZE_CASES
    got = wf.batch([c[1].encode() for c in SERIALIZE_CASES], True)
    for (name, body, _, _, _, err), (st_, _, a, k, _, _) in zip(SERIALIZE_CASES, got):
        if err:
            assert st_ == REJECTED, name
            continue
        assert st_ == OK and (a, k) == go_record_values(body.encode(), True), (name, a, k)
    assert [g[3] for g in got[:6]] == [b"{}", b"{}", b'{"mykwarg":1,"mykwarg2":2}', b'{"mykwarg":"value"}', b"{}", b'{"test":1}']


# ---------------------------------------------------------------------------------------------- named edges
def test_go_text_of_numbers(wf):
    for lit, want in (("1.0", "1"), ("1e2", "100"), ("-0", "-0"), ("-0.0", "-0"), ("1e-7", "1e-7"), ("1e21", "1e+21"),
                      ("12345678901234567890", "12345678901234567000"), ("1E3", "1000"), ("1.5", "1.5"), ("9007199254740993", "9007199254740992"),
                      ("0.000001", "0.000001"), ("1e-6", "0.000001"), ("123456789e15", "1.23456789e+23"), ("1e20", "100000000000000000000")):
        (st_, _, a, _, _, _), = wf.batch([b'{"args": [' + lit.encode() + b"]}"], False)
        assert st_ == OK and a == ("[" + want + "]").encode(), (lit, a)


KEY_CASES = [
    # equal only after unescaping: duplicates, the last one wins
    '{"a": 1, "\\u0061": 2}', '{"\\u00e9": 1, "é": 2}', '{"/": 1, "\\/": 2}', '{"a\\u0000": 1, "a": 2, "a\\u0000": 3}',
    # invalid UTF-8 and lone surrogates are U+FFFD: all one key
    '{"\\ud800": 1, "\\udfff": 2}', '{"\\ufffd": 1, "\\ud800": 2}', '{"\\udbff": 1, "\\ufffd": 2, "z": 0}',
    '{"x\\ud800y": 1, "x\\ufffdy": 2, "x": 3}',
    # UTF-8 byte order differs from UTF-16 order
    '{"\\uffff": 1, "\\ud83d\\ude00": 2}', '{"\\ud83d\\ude00": 1, "\\uffff": 2}', '{"\\ue000": 1, "\\ud800\\udc00": 2, "\\uff61": 3}',
    '{"a\\uffff": 1, "a\\ud83d\\ude00": 2, "a": 3, "a\\u007f": 4, "a\\u0080": 5}',
    # HTML-safe escaping in keys and values of a reordered object
    '{"b": "<", "a": "&", "c>": "\\u2028"}',
]
RAW_KEY_CASES = [b'{"\xff": 1, "\xfe": 2, "\xef\xbf\xbd": 3}', b'{"a\xc3": 1, "a\\ufffd": 2}', b'{"\xed\xa0\x80": 1, "\\ud800": 2, "b": 0}',
                 b'{"z": 1, "\xf4\x90\x80\x80": 2, "\xc0\x80": 3}']


@pytest.mark.parametrize("http", [False, True], ids=["sdk_payload", "http_body"])
def test_key_order_and_duplicates(wf, http):
    docs = [d.encode() for d in KEY_CASES] + RAW_KEY_CASES
    payloads = []
    for d in docs:
        payloads += [b'{"args": [' + d + b'], "kwargs": ' + d + b"}", b'{"kwargs": ' + d + b', "args": [1.5]}', d]
    answered, declined = check(wf, payloads, http, min_answered=1.0)
    assert declined == 0


@pytest.mark.parametrize("http", [False, True], ids=["sdk_payload", "http_body"])
def test_depth_and_member_limits(wf, http):
    """the walk answers 16 levels and 64 members and declines 17 / 65 (leaves of 1.5: go_transcode declines them all)"""
    cases = []                                            # (payload, answered?)
    for depth in (15, 16, 17):
        for objs in ((), tuple(range(0, depth, 2)), tuple(range(depth))):
            inner = _nest(depth - 1, "1.5", tuple(d - 1 for d in objs if d > 0))     # args / kwargs itself is level 1
            cases.append((b'{"args": [' + inner.encode() + b"]}", depth <= 16))
            if http:                                      # a body's remaining map: the body is level 1
                cases.append((('{"x": ' + inner + "}").encode(), depth <= 16))
    for n in (63, 64, 65):
        w = _wide(n, lambda i: "%d.5" % (n - i))
        cases.append((b'{"args": [], "kwargs": ' + w.encode() + b"}", n <= 64))
        cases.append((b'{"args": [1, ' + w.encode() + b"]}", n <= 64))
        if http:
            cases.append((w.encode(), n <= 64))
    got = wf.batch([c[0] for c in cases], http)
    for (p, ok), (st_, _, a, k, _, _) in zip(cases, got):
        if ok:
            assert st_ == OK and (a, k) == go_record_values(p, http), (p[:80], st_)
        else:
            assert st_ == UNSUPPORTED, p[:80]


def test_transcode_and_walk_agree_on_canonical_values(wf):
    """go_transcode's domain (sorted keys, short integers) through the walk gives the same bytes, white space or not"""
    rng = np.random.default_rng(7)
    toks = []
    for _ in range(3000):
        v = _random_value(random.Random(int(rng.integers(1 << 30))), 3, floats=False)
        for t in (json.dumps([v], sort_keys=True), json.dumps([v], sort_keys=True, separators=(",", ":"), ensure_ascii=False)):
            toks.append(t.encode())
    same = 0
    for t in toks:
        tr = wf.transcode(t)
        if tr is not None:
            assert wf.walk(t) == tr, t
            same += 1
    assert same > len(toks) // 2


# ---------------------------------------------------------------------------------------------- hypothesis
def _random_value(r: random.Random, depth: int, floats: bool = True):
    k = r.randrange(8 if depth else 5)
    if k == 0:
        return None
    if k == 1:
        return r.random() < 0.5
    if k == 2:
        return r.randrange(-10 ** 6, 10 ** 6)
    if k == 3:
        return "".join(r.choice('ab<>&"\\\n\x01é😀 ') for _ in range(r.randrange(4)))
    if k == 4:
        return r.uniform(-1e3, 1e3) if floats else r.randrange(100)
    if k in (5, 6):
        return {"".join(r.choice("abcé😀<") for _ in range(r.randrange(3))): _random_value(r, depth - 1, floats)
                for _ in range(r.randrange(5))}
    return [_random_value(r, depth - 1, floats) for _ in range(r.randrange(4))]


def _spell_number(x, r: random.Random) -> str:
    if isinstance(x, int):
        return r.choice([str(x), "%d.0" % x, "%de0" % x, "%d.000E+0" % x])
    return r.choice([repr(x), "%.17g" % x, "%.20e" % x])


def _dump_shuffled(v, r: random.Random) -> str:
    """JSON text of v with members in a random order, random earlier duplicates of some keys, random escapes / spacing"""
    ws = r.choice(["", " ", "\n\t"])
    if isinstance(v, dict):
        items = [(k, _dump_shuffled(x, r)) for k, x in v.items()]
        r.shuffle(items)
        out = []
        for key, text in items:
            if r.random() < 0.3:                          # an earlier duplicate: the later one wins
                out.append((key, _dump_shuffled(_random_value(r, 1), r)))
            out.append((key, text))
        return "{" + ws + ("," + ws).join(json.dumps(kk, ensure_ascii=r.random() < 0.5) + ws + ":" + ws + t for kk, t in out) + ws + "}"
    if isinstance(v, list):
        return "[" + ws + ("," + ws).join(_dump_shuffled(x, r) for x in v) + ws + "]"
    if isinstance(v, bool) or v is None:
        return json.dumps(v)
    if isinstance(v, (int, float)):
        return _spell_number(v, r)
    return json.dumps(v, ensure_ascii=r.random() < 0.5)


@settings(max_examples=400, deadline=None, suppress_health_check=list(HealthCheck))
@given(st.integers(0, 2 ** 32 - 1))
def test_shuffled_dicts_with_duplicates(wf, seed):
    r = random.Random(seed)
    args = [_random_value(r, 3) for _ in range(r.randrange(3))]
    kwargs = {"k%d" % i: _random_value(r, 3) for i in range(r.randrange(4))}
    body = {"a%d" % i: _random_value(r, 2) for i in range(r.randrange(4))}
    if r.random() < 0.5:
        body["args"] = args
    sdk = '{"kwargs": ' + _dump_shuffled(kwargs, r) + ', "args": ' + _dump_shuffled(args, r) + "}"
    http = _dump_shuffled(body, r)
    for payload, is_http in ((sdk, False), (sdk, True), (http, True), (http, False)):
        check(wf, [payload.encode()], is_http, min_answered=0.0)
