"""The endpoint drain's sequential half on a CPU (b9_endpoint_drain_launch): endpoint_device.cuh compiled for the host by
tests/host_shim/endpoint_shim.cpp, against the oracle's endpoint request (oracle/pyoracle/endpoint.py), which is itself
pinned by the reference's own EndpointManager (tests/golden/ref_endpoint_golden.json). Whatever the oracle answers 200,
400 or 500-from-the-handler, the build answers the same, byte for byte; each of its UNSUPPORTED carries one of the
documented reasons (`declined`)."""
import base64
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

from oracle.pyoracle import endpoint as EP

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_shim", "endpoint_shim.cpp")
SO = os.path.join(HERE, "host_shim", "libendpointshim.so")
GXX = os.environ.get("CXX", "g++")
HANDLERS = ["identity", "crc32", "vadd_f32", "json_sum"]
COMPLETE, ERROR, REJECTED, UNSUPPORTED = 0, 1, 3, 4
TF_HTTP_BODY = 0x02
GOLDEN = os.path.join(HERE, "golden", "ref_endpoint_golden.json")


def golden_cases():
    g = json.load(open(GOLDEN))
    return [(base64.b64decode(c["body"]), c["results"]) for c in g["cases"]]


@pytest.fixture(scope="module")
def ep():
    csrc = os.path.join(os.path.dirname(HERE), "beta9_b200", "csrc")
    deps = [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".h"))]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max([os.path.getmtime(SRC)] + [os.path.getmtime(d) for d in deps]):
        r = subprocess.run([GXX, "-O2", "-std=c++17", "-shared", "-fPIC", "-o", SO, SRC], capture_output=True, text=True)
        if r.returncode:
            pytest.skip("no host C++ compiler for the shim: " + r.stderr[-300:])
    lib = C.CDLL(SO)
    u64p, u8p = np.ctypeslib.ndpointer(np.uint64, flags="C"), np.ctypeslib.ndpointer(np.uint8, flags="C")
    lib.b9_ep_batch.argtypes = [C.c_char_p, u64p, u8p, C.c_uint32, C.c_int, u8p, u8p, C.c_void_p, u64p]
    lib.b9_ep_batch.restype = C.c_uint64

    def batch(bodies, handler, flags=TF_HTTP_BODY):
        """[(status, has, record bytes)] per body"""
        n = len(bodies)
        off = np.zeros(n + 1, np.uint64)
        np.cumsum([len(b) for b in bodies], out=off[1:])
        blob = b"".join(bodies) + b"\0" * 8
        fl = np.full(max(n, 1), flags, np.uint8)
        status, has, out_off = np.zeros(max(n, 1), np.uint8), np.zeros(max(n, 1), np.uint8), np.zeros(n + 1, np.uint64)
        total = lib.b9_ep_batch(blob, off, fl, n, HANDLERS.index(handler), status, has, None, out_off)
        out = np.zeros(total + 1, np.uint8)
        lib.b9_ep_batch(blob, off, fl, n, HANDLERS.index(handler), status, has, out.ctypes.data, out_off)
        raw = out.tobytes()
        return [(int(status[i]), int(has[i]), raw[int(out_off[i]):int(out_off[i + 1])]) for i in range(n)]
    return batch


def as_outcome(status, has, data):
    """a device record as the oracle's (outcome, bytes)"""
    if status == COMPLETE:
        assert has == 1
        return EP.OK, data
    assert has == 0 and data == b""
    if status == REJECTED:
        return EP.BAD_REQUEST, EP.INVALID_PAYLOAD_BODY
    if status == ERROR:
        return EP.HANDLER_RAISED, None
    return "UNSUPPORTED", None


def _literals(body):
    """(number literals, max nesting, max members of an object) of the body as json.loads reads it, or None"""
    nums, depth, members = [], [0], [0]
    try:
        text = body.decode("utf-8", "replace")
    except Exception:
        return None

    def num(s):
        nums.append(s)
        return 0

    def pairs(kv):
        members[0] = max(members[0], len(kv))
        return dict(kv)
    try:
        doc = json.loads(text, parse_float=num, parse_int=num, object_pairs_hook=pairs)
    except (ValueError, RecursionError):
        return None

    def walk(v, d):
        depth[0] = max(depth[0], d)
        if isinstance(v, dict):
            for x in v.values():
                walk(x, d + 1)
        elif isinstance(v, list):
            for x in v:
                walk(x, d + 1)
    walk(doc, 0)
    return nums, depth[0], members[0]


def _sig_digits(lit):
    m = lit.lstrip("-").split("e")[0].split("E")[0].replace(".", "").lstrip("0")
    return len(m.rstrip("0")) if m else 0


def declined(body, handler):
    """The documented reasons for an endpoint drain's UNSUPPORTED (include/b9gpu.h, b9_endpoint_drain_launch): a render
    failure (json_sum's non-finite total), a number of more than 19 significant digits, nesting deeper than 16, an
    object of more than 64 members, a json_sum int outside a C long, vadd_f32's escaped base64 alphabet."""
    outcome, _ = EP.run_endpoint_request(body, handler)
    if outcome == EP.RENDER_FAILED:
        return True
    lit = _literals(body)
    if lit is None:
        return False
    nums, depth, members = lit
    if any(_sig_digits(x) > 19 for x in nums) or depth > 16 + 2 or members > 64:
        return True
    if handler == "json_sum" and any(abs(int(x)) >= 2**62 for x in nums if all(ch not in x for ch in ".eE")) or \
       handler == "json_sum" and any(abs(float(x)) >= 2**62 for x in nums):
        return True
    if handler == "vadd_f32" and b"\\" in body:
        return True
    return False


def check(ep, bodies, handler, want=None):
    """want: the oracle's (outcome, bytes) per body (computed when None). Returns the number of answered bodies."""
    answered = 0
    for i, (b, got) in enumerate(zip(bodies, ep(bodies, handler))):
        g = as_outcome(*got)
        if g[0] == "UNSUPPORTED":
            assert declined(b, handler), (handler, b[:160])
            continue
        w = want[i] if want is not None else EP.run_endpoint_request(b, handler)
        assert g == w, (handler, b[:160], g, w)
        answered += 1
    return answered


def _golden_want(r):
    if r["status_code"] == 400:
        return EP.BAD_REQUEST, EP.INVALID_PAYLOAD_BODY
    if r["status_code"] == 200:
        return EP.OK, base64.b64decode(r["body"])
    return (EP.HANDLER_RAISED if r["task_status"] == "ERROR" else EP.RENDER_FAILED), None


@pytest.mark.parametrize("handler", HANDLERS)
def test_oracle_equals_the_reference_golden(handler):
    cases = golden_cases()
    assert len(cases) > 500
    for body, res in cases:
        assert EP.run_endpoint_request(body, handler) == _golden_want(res[handler]), (handler, body[:120])


@pytest.mark.parametrize("handler", HANDLERS)
def test_device_build_answers_the_golden(ep, handler):
    cases = golden_cases()
    bodies = [b for b, _ in cases]
    want = [_golden_want(r[handler]) for _, r in cases]
    answered = check(ep, bodies, handler, want)
    assert answered >= len(bodies) - 12, answered


def test_golden_renders_what_the_issue_names(ep):
    """the rendering differences from the task-queue result, spelled out"""
    one = lambda v, h="identity": ep([b'{"args": [' + v + b']}'], h)[0]     # noqa: E731
    assert one(b'"\xc3\xa9"') == (COMPLETE, 1, b'"\xc3\xa9"')
    assert one(b'"\\u00e9"') == (COMPLETE, 1, b'"\xc3\xa9"')
    assert one(b'[1, "a"]') == (COMPLETE, 1, b'[1,"a"]')
    for v, r in ((b'""', b'""'), (b'0', b'0'), (b'-0', b'0'), (b'-0.0', b'0'), (b'null', b'null'), (b'false', b'false'),
                 (b'[]', b'[]'), (b'{}', b'{}'), (b'1.0', b'1'), (b'1e21', b'1e+21'), (b'"\\u2028<\x7f"', b'"\xe2\x80\xa8<\x7f"'),
                 (b'"\\ud800"', b'"\xef\xbf\xbd"'), (b'"\xff"', b'"\xef\xbf\xbd"'), (b'"\\u001f\\n"', b'"\\u001f\\n"')):
        assert one(v) == (COMPLETE, 1, r), v
    assert one(b'""', "crc32") == (COMPLETE, 1, b"0")
    assert one(b'""', "vadd_f32") == (COMPLETE, 1, b'""')
    assert one(b'{"values": [0]}', "json_sum") == (COMPLETE, 1, b"0")
    assert one(b'{"values": [0.5, -0.5]}', "json_sum") == (COMPLETE, 1, b"0.0")
    assert one(b'{"values": [1e308, 1e308]}', "json_sum")[0] == UNSUPPORTED


@pytest.mark.parametrize("handler", HANDLERS)
def test_only_plain_http_bodies_are_answered(ep, handler):
    body = b'{"args": ["x"]}'
    for flags in (0x00, 0x04, 0x08, 0x02 | 0x04, 0x02 | 0x08):
        assert ep([body], handler, flags)[0] == (UNSUPPORTED, 0, b"")


@pytest.mark.parametrize("handler", HANDLERS)
def test_existing_http_and_parser_corpora(ep, handler):
    from tests.test_device_parser_on_host import _payloads
    from tests.test_gpu_parity import _http_bodies
    bodies = list(dict.fromkeys(list(_http_bodies()) + list(_payloads())))
    answered = check(ep, bodies, handler)
    assert answered > len(bodies) * 9 // 10


_json = st.recursive(
    st.none() | st.booleans() | st.integers(min_value=-2**70, max_value=2**70)
    | st.floats(allow_nan=False, allow_infinity=False) | st.text(max_size=12),
    lambda kids: st.lists(kids, max_size=5) | st.dictionaries(st.text(max_size=6), kids, max_size=5),
    max_leaves=20)


@settings(max_examples=400, deadline=None, suppress_health_check=list(HealthCheck))
@given(v=_json, ascii_=st.booleans())
def test_hypothesis_documents(ep, v, ascii_):
    bodies = [json.dumps({"args": [v]}, ensure_ascii=ascii_).encode("utf-8", "surrogatepass"),
              json.dumps({"args": [{"values": v if isinstance(v, list) else [v]}]}).encode("utf-8", "surrogatepass")]
    if isinstance(v, dict):
        bodies.append(json.dumps(v, ensure_ascii=ascii_).encode("utf-8", "surrogatepass"))
    for h in HANDLERS:
        check(ep, bodies, h)


@pytest.mark.parametrize("handler", HANDLERS)
def test_single_byte_mutations(ep, handler):
    """30 k bodies with one byte replaced, deleted or inserted, over the golden's and the synthetic bodies"""
    from beta9_b200 import synth
    base = [b for b, _ in golden_cases() if len(b) >= 4]
    for bt in (synth.json_batch(8, doc_bytes=200), synth.vadd_batch(8, floats_per_vec=3), synth.strings_batch(40, 48, adversarial_frac=0.4, seed=5)):
        base += [bt.task(i) for i in range(bt.n)]
    rng = np.random.default_rng(7 + HANDLERS.index(handler))
    alphabet = list(b'{}[],:" 01e.-nulltrackwgsAv\\\x7f') + [0xC3, 0xA9, 0xFF, 0x1F]
    bodies = []
    while len(bodies) < 30000 // len(HANDLERS):
        b = base[int(rng.integers(0, len(base)))]
        m = bytearray(b)
        pos = int(rng.integers(0, len(m)))
        op = int(rng.integers(0, 3))
        ch = int(rng.choice(alphabet))
        if op == 0: m[pos] = ch
        elif op == 1: del m[pos]
        else: m[pos:pos] = bytes([ch])
        bodies.append(bytes(m))
    check(ep, bodies, handler)


def test_non_finite_sums_are_declined_not_rendered(ep):
    for vals in (b'[1e308, 1e308]', b'[-1e308, -1e308]', b'[1e308, 1e308, -1e308]'):
        body = b'{"args": [{"values": ' + vals + b'}]}'
        assert EP.run_endpoint_request(body, "json_sum")[0] == EP.RENDER_FAILED
        assert ep([body], "json_sum")[0] == (UNSUPPORTED, 0, b"")
    assert math.isinf(sum([1e308, 1e308]))
