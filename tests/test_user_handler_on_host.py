"""User handlers on a CPU: the generic half of the user-handler drain (include/b9gpu_handler.cuh: the parse each rendering
accepts, phase A with the counting sink, phase B with the writing sink) and the example handlers
(examples/handlers/handlers.cuh), compiled for the host by tests/host_shim/user_handler_shim.cpp, against their Python
twins (examples/handlers/handlers.py) run through the oracle's loops: the task-queue loop over SDK payloads and HTTP
bodies, the runner's half over TaskMessage records, and the endpoint request. Statuses, has_result, record bytes and the
exception class of every ERROR must agree; an UNSUPPORTED must carry one of the documented reasons (`may_decline`).
echo_str and crc32_str must also equal the built-in identity and crc32 host builds wherever the argument is a str."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from oracle.pyoracle import endpoint as EP
from oracle.pyoracle.gojson import GoJSONError, go_unmarshal_task_payload
from oracle.pyoracle.httpserialize import InvalidRequestPayload
from oracle.pyoracle.loop import run_task_loop
from oracle.pyoracle.wire import QueueEnv, build_task_message, format_uuid
from tests.task_msg_oracle import NOT_RUN, run_records

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "examples", "handlers"))
import handlers as twins  # noqa: E402  (examples/handlers/handlers.py)

SRC = os.path.join(HERE, "host_shim", "user_handler_shim.cpp")
SO = os.path.join(HERE, "host_shim", "libuserhandlershim.so")
GXX = os.environ.get("CXX", "g++")
NAMES = ["echo_str", "crc32_str", "word_count", "prod"]
COMPLETE, ERROR, REJECTED, UNSUPPORTED = 0, 1, 3, 4
TF_HTTP_BODY, TF_TASK_MSG = 0x02, 0x08
EXC = {TypeError: 0x01, AttributeError: 0x02, UnicodeEncodeError: 0x04, KeyError: 0x08, ValueError: 0x10}
TQ, ENDPOINT = 0, 1


def _deps():
    out = [SRC, os.path.join(ROOT, "include", "b9gpu_handler.cuh"), os.path.join(ROOT, "include", "b9gpu.h"),
           os.path.join(ROOT, "examples", "handlers", "handlers.cuh")]
    csrc = os.path.join(ROOT, "beta9_b200", "csrc")
    return out + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".h"))]


def _shim(src, so, extra=()):
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in _deps() + [src]):
        r = subprocess.run([GXX, "-O2", "-std=c++17", "-shared", "-fPIC", *extra, "-o", so, src], capture_output=True, text=True)
        if r.returncode:
            pytest.skip("no host C++ compiler for the shim: " + r.stderr[-300:])
    return C.CDLL(so)


@pytest.fixture(scope="module")
def uh():
    lib = _shim(SRC, SO, ["-I" + os.path.join(ROOT, "include")])
    u64p, u8p, i64p = (np.ctypeslib.ndpointer(t, flags="C") for t in (np.uint64, np.uint8, np.int64))
    lib.b9_uh_batch.argtypes = [C.c_char_p, u64p, u8p, u8p, C.c_uint32, C.c_int, C.c_int, u8p, u8p, i64p, C.c_void_p, u64p]
    lib.b9_uh_batch.restype = C.c_uint64

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
        total = lib.b9_uh_batch(blob, off, fl, idb, n, h, rendering, status, has, val, None, out_off)
        out = np.zeros(total + 1, np.uint8)
        lib.b9_uh_batch(blob, off, fl, idb, n, h, rendering, status, has, val, out.ctypes.data, out_off)
        raw = out.tobytes()
        return [(int(status[i]), int(has[i]), int(val[i]), raw[int(out_off[i]):int(out_off[i + 1])]) for i in range(n)]
    return batch


# ---- when may the device decline? -------------------------------------------------------------------------------------
def _long_literal(body: bytes) -> bool:
    """a number literal of more than 15 significant digits (f64_parse may not settle those past 19) or nesting past 64"""
    import re
    if body.count(b"[") + body.count(b"{") > 60:
        return True
    return any(len(m.replace(b".", b"").lstrip(b"0")) > 15 for m in re.findall(rb"[0-9][0-9.]*", body))


def _prod_overflows(xs) -> bool:
    if not isinstance(xs, list):
        return False
    p = 1
    for x in xs:
        if type(x) not in (int, float, bool):
            return False
        if type(x) is int and not -2**63 <= x < 2**63:
            return True
        p *= x
        if type(p) is int and not -2**63 <= p < 2**63:
            return True
    return False


def may_decline(name, payload, args):
    if _long_literal(payload):
        return True
    return name == "prod" and args is not None and len(args) == 1 and _prod_overflows(args[0])


def exc_bit(fn, args, kwargs):
    if len(args) != 1 or kwargs:
        return EXC[TypeError]
    try:
        fn(*args)
    except BaseException as e:              # noqa: BLE001
        return EXC.get(type(e), -1)
    return 0


# ---- the comparisons ---------------------------------------------------------------------------------------------------
def check_tq(uh, name, payloads, http=False):
    """The task-queue rendering against run_task_loop. Returns the number of tasks the device answered."""
    fn = twins.TWINS[name]
    ids = [i.to_bytes(16, "little") for i in range(len(payloads))]
    want = run_task_loop(payloads, ids, handler=fn, http_body=http, keep_wire=True)
    got = uh(payloads, name, TQ, TF_HTTP_BODY if http else 0)
    answered = 0
    for p, w, (st_, has, val, data) in zip(payloads, want, got):
        args = kwargs = None
        if w.wire is not None:
            t = json.loads(w.wire)
            args, kwargs = t["args"] or [], t["kwargs"] or {}
        if st_ == UNSUPPORTED:
            assert may_decline(name, p, args), (name, p, w)
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


def check_ep(uh, name, bodies):
    fn = twins.TWINS[name]
    got = uh(bodies, name, ENDPOINT, TF_HTTP_BODY)
    answered = 0
    for b, (st_, has, _, data) in zip(bodies, got):
        outcome, want = EP.run_endpoint_request(b, fn)
        if st_ == UNSUPPORTED:
            try:
                args = json.loads(EP.gateway_body(b))["args"]
            except (InvalidRequestPayload, GoJSONError, ValueError, RecursionError):
                args = None
            assert outcome == EP.RENDER_FAILED or may_decline(name, b, args), (name, b, outcome)
            continue
        answered += 1
        if st_ == COMPLETE:
            assert (outcome, data) == (EP.OK, want) and has == 1, (name, b, outcome, want, data)
        elif st_ == REJECTED:
            assert outcome == EP.BAD_REQUEST and has == 0, (name, b, outcome)
        else:
            assert st_ == ERROR and outcome == EP.HANDLER_RAISED and has == 0, (name, b, outcome, st_)
    return answered


def records_of(payloads):
    """TaskMessage records of the payloads Go accepts, with the ids they carry"""
    recs, ids = [], []
    for i, p in enumerate(payloads):
        try:
            args, kwargs = go_unmarshal_task_payload(p)
        except GoJSONError:
            continue
        tid = (i + 1).to_bytes(16, "big")
        recs.append(build_task_message(QueueEnv(), format_uuid(tid), args, kwargs, 1_789_970_992_573_161_412).encode())
        ids.append(tid)
    return recs, ids


def check_records(uh, name, records, ids):
    fn = twins.TWINS[name]
    want = run_records(records, ids, fn)
    got = uh(records, name, TQ, TF_TASK_MSG, ids)
    answered = 0
    for r, w, (st_, has, val, data) in zip(records, want, got):
        if st_ == UNSUPPORTED:
            args = json.loads(r)["args"] if w.status != NOT_RUN else None
            assert w.status == NOT_RUN or may_decline(name, r, args), (name, r, w)
            continue
        answered += 1
        assert st_ == {"COMPLETE": COMPLETE, "ERROR": ERROR}[w.status], (name, r, w)
        assert (has, data if has else None) == (1 if w.result is not None else 0, w.result), (name, r, w.result, data)
    return answered


# ---- corpora -------------------------------------------------------------------------------------------------------------
def sdk(*args, **kwargs):
    return json.dumps({"args": args, "kwargs": kwargs}).encode()


SPACES = "\t\n\x0b\x0c\r\x1c\x1d\x1e\x1f \x85\xa0        　"
HANDMADE = [sdk(s) for s in ["", "a", "hello world", "  a  b  ", SPACES, "x" + SPACES + "y", "​", "café \U0001F600",
                             "\ud800", "a\"b\\c\n\x00\x7f", "\x1c\x1d", "᠎"]] + \
    [sdk(v) for v in [None, True, False, 0, 1, -1, 1.5, -0.0, [], {}, [1, 2, 3], [2, 0.5], [True, 3], [1e308, 10.0],
                      [1e308, 10.0, 0.0], [2**40, 2**40], [-2**62, 2], [-2**62, 2, -1], [1, "a"], [[1]], {"a": 1}, [None],
                      [0.1, 0.2, 0.3], [3, 1e-320], [float("nan")] if False else [7]]] + \
    [sdk("a", "b"), sdk(), sdk("a", k=1), b'{"args": ["a"], "kwargs": null}', b'{"args": null}', b'not json', b'{"args": [1e400]}',
     b'{"args": [[1e400]]}', b'{"args": [12345678901234567890123]}', b'{"args": [[12345678901234567890123, 2]]}',
     b'{"args": [[1.00000000000000011102230246251565404236316680908203125]]}', b'{"args": ["\\ud800\\udc00"]}',
     b'{"args": ["\\udc00x"]}', b'{"args": ["\xff\xfe"]}', b'{"args": [-0]}', b'{"args": [[-0, 5]]}', b'{"args": [1e21]}',
     b'{"args": [[1e20, 10]]}', b'{"args": [[1E2, 3]]}']


def golden_payloads():
    from tests import golden_util
    import base64
    out = []
    for cases in golden_util.load()["groups"].values():
        out += [base64.b64decode(c["payload"]) for c in cases]
    return out


def corpus():
    from tests.test_device_parser_on_host import _payloads
    from tests.test_gpu_parity import _http_bodies
    return list(dict.fromkeys(HANDMADE + golden_payloads() + list(_payloads()) + list(_http_bodies())))


# ---- tests ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_sdk_payloads_and_http_bodies(uh, name):
    c = corpus()
    assert check_tq(uh, name, c) > len(c) * 9 // 10
    assert check_tq(uh, name, c, http=True) > len(c) * 8 // 10
    assert check_ep(uh, name, c) > len(c) * 8 // 10


@pytest.mark.parametrize("name", NAMES)
def test_task_message_records(uh, name):
    recs, ids = records_of(corpus())
    assert check_records(uh, name, recs, ids) > len(recs) * 9 // 10
    # records only: an HTTP body or a pickle flag beside the record flag, and a record of another id, are not answered
    assert all(g[0] == UNSUPPORTED for g in uh(recs[:50], name, TQ, TF_TASK_MSG | TF_HTTP_BODY, ids[:50]))
    assert all(g[0] == UNSUPPORTED for g in uh(recs[:50], name, TQ, TF_TASK_MSG, ids[1:51]))


@pytest.mark.parametrize("name", NAMES)
def test_pickle_and_foreign_flags_are_unsupported(uh, name):
    ps = [sdk("a"), sdk([1, 2])]
    for fl in (0x04, 0x04 | 0x02):
        assert all(g[0] == UNSUPPORTED for g in uh(ps, name, TQ, fl))
    for fl in (0, 0x04, 0x08):
        assert all(g[0] == UNSUPPORTED for g in uh(ps, name, ENDPOINT, fl))


def test_f64_corpus(uh):
    from tests.f64_corpus import _literals
    rng = np.random.default_rng(11)
    lits = _literals()
    pick = [lits[i] for i in rng.choice(len(lits), 6000, replace=False)]
    bodies = [b'{"args": [[%s]]}' % s.encode() for s in pick] + [b'{"args": [[%s, 3, 0.5]]}' % s.encode() for s in pick[:2000]] + \
             [b'{"args": [%s]}' % s.encode() for s in pick[:2000]]
    for name in NAMES:
        check_tq(uh, name, bodies)
        check_ep(uh, name, bodies)
    recs, ids = records_of(bodies[:3000])
    check_records(uh, "prod", recs, ids)


_cp = st.characters(min_codepoint=0, max_codepoint=0x10FFFF)
_space = st.sampled_from(list(SPACES) + [" ", "a", "​", "᠎"])
_num = st.integers(min_value=-2**66, max_value=2**66) | st.floats() | st.booleans() | st.sampled_from([0, -0.0, 1, 2**63 - 1, -2**63])
_arg = st.text(_cp, max_size=20) | st.text(_space, max_size=12) | st.lists(_num, max_size=8) | \
    st.lists(_num | st.text(max_size=3) | st.none(), max_size=4) | _num | st.none() | st.dictionaries(st.text(max_size=3), _num, max_size=2)


@settings(max_examples=500, deadline=None, suppress_health_check=list(HealthCheck))
@given(v=_arg, ascii_=st.booleans())
def test_hypothesis_values(uh, v, ascii_):
    try:
        body = json.dumps({"args": [v], "kwargs": {}}, ensure_ascii=ascii_).encode("utf-8", "surrogatepass")
    except ValueError:
        return
    for name in NAMES:
        check_tq(uh, name, [body])
        check_tq(uh, name, [body], http=True)
        check_ep(uh, name, [body])
        recs, ids = records_of([body])
        check_records(uh, name, recs, ids)


@pytest.mark.parametrize("name", NAMES)
def test_single_byte_mutations(uh, name):
    """30 k payloads with one byte replaced, deleted or inserted"""
    base = [b for b in corpus() if len(b) >= 4][:400] + [sdk("w o r d s　x"), sdk([2, 3.5, True]), sdk([1, 2, 3, 4, 5, 6])]
    rng = np.random.default_rng(31 + NAMES.index(name))
    alphabet = list(b'{}[],:" 01e.-nulltrackwgsAv\\\x7f\t') + [0xC3, 0xA9, 0xFF, 0x1F, 0xE3, 0x80]
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
    check_tq(uh, name, bodies)
    check_ep(uh, name, bodies)


def test_echo_and_crc32_equal_the_built_in_host_builds(uh):
    """str arguments: echo_str's records are identity's and crc32_str's are crc32's, byte for byte, in both renderings"""
    hp = _shim(os.path.join(HERE, "host_shim", "host_parse.cpp"), os.path.join(HERE, "host_shim", "libhostparse_uh.so"))
    hp.b9_host_run.argtypes = [C.c_char_p, C.c_uint32, C.c_int, C.c_int, C.POINTER(C.c_uint8), C.POINTER(C.c_uint8), C.c_void_p, C.c_uint32]
    hp.b9_host_run.restype = C.c_long
    ep = _shim(os.path.join(HERE, "host_shim", "endpoint_shim.cpp"), os.path.join(HERE, "host_shim", "libendpointshim_uh.so"))
    u64p, u8p = np.ctypeslib.ndpointer(np.uint64, flags="C"), np.ctypeslib.ndpointer(np.uint8, flags="C")
    ep.b9_ep_batch.argtypes = [C.c_char_p, u64p, u8p, C.c_uint32, C.c_int, u8p, u8p, C.c_void_p, u64p]
    ep.b9_ep_batch.restype = C.c_uint64
    rng = np.random.default_rng(3)
    strs = ["", "a", "café", "\ud800", "\U0001F600x", "tab\tquote\"back\\", "\x00\x1f\x7f", SPACES]
    for _ in range(3000):
        cps = rng.integers(0, 0x110000, size=int(rng.integers(0, 30)))
        strs.append("".join(chr(int(c)) if rng.random() < 0.5 else chr(int(c) % 128) for c in cps))
    payloads = []
    for s in strs:
        for asc in (True, False):
            payloads.append(json.dumps({"args": [s], "kwargs": {}}, ensure_ascii=asc).encode("utf-8", "surrogatepass"))
    for http in (0, 1):
        for name, builtin in (("echo_str", 0), ("crc32_str", 1)):
            got = uh(payloads, name, TQ, TF_HTTP_BODY if http else 0)
            for p, (st_, has, _, data) in zip(payloads, got):
                s_, h_ = C.c_uint8(), C.c_uint8()
                buf = (C.c_uint8 * (len(p) * 12 + 64))()
                n = hp.b9_host_run(p, len(p), http, builtin, C.byref(s_), C.byref(h_), buf, len(buf))
                assert (st_, has, data) == (s_.value, h_.value, bytes(buf[:max(n, 0)]) if h_.value else b""), (name, p)
    for name, builtin in (("echo_str", 0), ("crc32_str", 1)):
        got = uh(payloads, name, ENDPOINT, TF_HTTP_BODY)
        n = len(payloads)
        off = np.zeros(n + 1, np.uint64)
        np.cumsum([len(b) for b in payloads], out=off[1:])
        blob = b"".join(payloads) + b"\0" * 8
        fl = np.full(n, TF_HTTP_BODY, np.uint8)
        status, has, out_off = np.zeros(n, np.uint8), np.zeros(n, np.uint8), np.zeros(n + 1, np.uint64)
        total = ep.b9_ep_batch(blob, off, fl, n, builtin, status, has, None, out_off)
        out = np.zeros(total + 1, np.uint8)
        ep.b9_ep_batch(blob, off, fl, n, builtin, status, has, out.ctypes.data, out_off)
        raw = out.tobytes()
        for i, (st_, h, _, data) in enumerate(got):
            assert (st_, h, data) == (status[i], has[i], raw[int(out_off[i]):int(out_off[i + 1])]), (name, payloads[i])


def test_two_passes_must_agree(uh):
    """the writing sink never writes past the reservation: a handler whose second pass differs is UNSUPPORTED (the shim
    reports 255 where phase B returned false); every example writes what it counted"""
    for name in NAMES:
        assert all(g[0] != 255 for g in uh(corpus(), name, TQ))


def test_example_cubin_exports_the_versioned_entries():
    """the cubin build() makes (compile_handlers: rebuilt only when a source is newer) is sm_90a and holds both entries
    of every example under the library's handler ABI version"""
    import shutil
    from beta9_b200 import build as B
    if not os.path.exists(B.NVCC):
        pytest.skip("no nvcc")
    out = B.build_examples()
    cuobjdump = shutil.which("cuobjdump") or os.path.join(os.path.dirname(B.NVCC), "cuobjdump")
    elf = subprocess.run([cuobjdump, "-elf", out], capture_output=True, text=True).stdout
    assert "sm_90a" in elf
    syms = subprocess.run([cuobjdump, "-symbols", out], capture_output=True, text=True).stdout
    v = B.handler_abi_version()
    for name in NAMES:
        for kind in ("tq", "ep"):
            assert f"b9h_v{v}_{kind}_{name}" in syms, (name, kind, syms[-2000:])
