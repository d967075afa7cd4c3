"""The function and endpoint runners' callbacks on a CPU: the device's writers (beta9_b200/csrc/callback_runners.cuh, built
for the host through tests/host_shim/callback_runners_shim.cpp) against json.dumps and the oracle's restatement
(tests/callback_runners_oracle.py: function_callback, endpoint_callback, endpoint_text)."""
import ctypes as C
import json
import os
import random
import subprocess

import cloudpickle
import pytest
from hypothesis import given, settings
from hypothesis import strategies as st

from oracle.pyoracle import callback as cb0
from tests import callback_runners_oracle as cb
from oracle.pyoracle import endpoint as EP
from oracle.pyoracle import funcloop
from tests.pickle_corpus import HANDLERS, frame_one, plain_values, structured_blobs

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_shim", "callback_runners_shim.cpp")
SO = os.path.join(HERE, "host_shim", "libcallback_runners.so")
GXX = os.environ.get("CXX", "g++")
CAP = 8 << 20
KIND = {0: cb.CB_POST, 1: cb.CB_UNSENDABLE, 2: cb.CB_HOST}


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(SRC), os.path.getmtime(
            os.path.join(HERE, "..", "beta9_b200", "csrc", "callback_runners.cuh"))):
        r = subprocess.run([GXX, "-O2", "-std=c++17", "-shared", "-fPIC", "-o", SO, SRC], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    lib = C.CDLL(SO)
    lib.b9_cbr_endpoint.restype = C.c_uint64
    lib.b9_cbr_endpoint.argtypes = [C.c_char_p, C.c_uint32, C.c_void_p]
    lib.b9_cbr_function.restype = C.c_int
    lib.b9_cbr_function.argtypes = [C.c_char_p, C.c_uint32, C.c_int, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    return lib


def device_endpoint(lib, e: bytes) -> bytes:
    n = lib.b9_cbr_endpoint(e, len(e), None)
    buf = C.create_string_buffer(max(1, n))
    assert lib.b9_cbr_endpoint(e, len(e), buf) == n
    return buf.raw[:n]


_BUF = None


def device_function(lib, blob: bytes, handler: str):
    """-> None (the pass does not complete the task), or (kind, D, url) as the function runner's callback pass settles it"""
    global _BUF
    if _BUF is None:
        _BUF = C.create_string_buffer(CAP)
    d, u = C.c_uint32(0), C.c_uint32(0)
    k = lib.b9_cbr_function(blob, len(blob), HANDLERS.index(handler), _BUF, CAP, C.byref(d), C.byref(u))
    assert k != -2
    if k == -1:
        return None
    kind = KIND[k]
    if kind != cb.CB_POST:
        return kind, None, None
    raw = _BUF.raw[:d.value + u.value]
    return kind, raw[:d.value], raw[d.value:].decode("utf-8") if u.value else None


def expected_function(blob: bytes, handler: str):
    status, res = funcloop.run_function_task(blob, handler)
    kwargs = funcloop.load_args(blob).get("kwargs") or {}
    return cb.function_callback(status, cloudpickle.loads(res) if status == "COMPLETE" else None, kwargs)


def check_function(lib, blob: bytes, handler: str) -> bool:
    got = device_function(lib, blob, handler)
    if got is None:
        return False
    assert got == expected_function(blob, handler), (blob, handler)
    return True


# ---------------------------------------------------------------------------------------------- 1. the oracle's D is json.dumps
def test_oracle_function_callback_rules():
    assert cb.function_callback("COMPLETE", None, {}) == (cb.CB_POST, b"null", None)
    assert cb.function_callback("COMPLETE", "", {"callback_url": "http://x"}) == (cb.CB_POST, b'""', "http://x")
    for falsy in (None, "", 0, b"", False):
        assert cb.function_callback("COMPLETE", 1, {"callback_url": falsy})[2] is None
    for bad in (b"http://x", 5, "\ud800x"):
        assert cb.function_callback("COMPLETE", 1, {"callback_url": bad})[0] == cb.CB_HOST
    assert cb.function_callback("COMPLETE", [1, b"x"], {})[0] == cb.CB_UNSENDABLE
    assert cb.function_callback("COMPLETE", {b"k": 1}, {})[0] == cb.CB_UNSENDABLE
    assert cb.function_callback("COMPLETE", {float("nan"): 1}, {})[0] == cb.CB_UNSENDABLE
    assert cb.function_callback("COMPLETE", [float("inf")], {})[0] == cb.CB_UNSENDABLE
    assert cb.function_callback("COMPLETE", [2 ** 63], {})[0] == cb.CB_HOST
    assert cb.function_callback("COMPLETE", {1: 2, 1.5: 3, None: 4, False: 5}, {})[1] == b'{"1": 2, "1.5": 3, "null": 4, "false": 5}'
    assert cb.function_callback("ERROR", None, {})[0] == cb.CB_HOST
    assert cb.endpoint_callback("REJECTED", None) == (cb.CB_NONE, None)
    assert cb.endpoint_callback("ERROR", None)[0] == cb.CB_HOST
    assert cb.endpoint_text('{"data":"\x7f\xe9\U0001F600"}'.encode()) == json.dumps({'data': '\x7f\xe9\U0001F600'}).encode()


# ---------------------------------------------------------------------------------------------- 2. function: D, URL and kind
@pytest.mark.parametrize("handler", HANDLERS)
def test_function_corpus(lib, handler):
    """Every structured blob of the pickle corpus (plain values, SDK documents, the goldens' blobs, hand-built graphs with
    shared members, callback_url kwargs): where the pass completes the task, the device's kind, D and URL are the oracle's."""
    blobs = structured_blobs()
    done = sum(check_function(lib, b, handler) for b in blobs)
    assert done > (len(blobs) // 3 if handler == "identity" else 20)


def test_function_callback_url_kwargs(lib):
    for url in (None, "", 0, "http://x", b"http://x", 5, "http://é/\U0001F600", "\ud800", False, [], ["u"]):
        blob = funcloop.frame_call("s", callback_url=url)
        got = device_function(lib, blob, "identity")
        assert got == expected_function(blob, "identity"), url


def test_function_values(lib):
    """Bytes results and keys, NaN / inf values and float keys, DEL and every UTF-8 length, lone surrogates, ints at the
    int64 edges and nested shared objects."""
    shared = {"k": ["é", 1.5]}
    vals = [b"x", [1, b""], {b"k": 1}, {"a": {b"k": 1}}, float("nan"), [float("inf")], {float("-inf"): 1}, {float("nan"): 1},
            {1.5: 1}, {-0.0: 1}, {2 ** 63 - 1: 1, -2 ** 63: 2}, {2 ** 63: 1}, 2 ** 63, -2 ** 63 - 1, "\x7f", "a\x00\x1f\"\\/\b\f\n\r\t",
            "é", "€", "\U0001F600", "\ud800", "\udfff", "x\ud83dy", [shared, shared, (shared,)], {"s": shared, "t": [shared]},
            (), (1,), [(), [], {}], None, True, False, {None: None, True: False, False: True}, 1e16, 1e-5, 1e22, -0.0, 5e-324]
    for v in vals + plain_values():
        check_function(lib, frame_one(v), "identity")


def test_function_code_points(lib):
    """Every code point class ensure_ascii distinguishes: the short escapes, the other C0 controls, DEL, ASCII, two-, three-
    and four-byte sequences, the surrogate range (lone, under surrogatepass) and the ends of each range."""
    cps = list(range(0x100)) + [0x7FF, 0x800, 0xFFF, 0x1000, 0xD7FF, 0xD800, 0xDBFF, 0xDC00, 0xDFFF, 0xE000, 0xFEFF, 0xFFFD,
                                 0xFFFE, 0xFFFF, 0x10000, 0x1F600, 0xFFFFF, 0x100000, 0x10FFFF, 0x2028, 0x2029]
    rng = random.Random(3)
    cps += [rng.randrange(0x110000) for _ in range(2000)]
    for k in range(0, len(cps), 64):
        s = "".join(chr(c) for c in cps[k:k + 64])
        got = device_function(lib, frame_one(s), "identity")
        assert got == (cb.CB_POST, json.dumps(s).encode(), None), s


_scalars = st.one_of(st.none(), st.booleans(), st.integers(min_value=-2 ** 70, max_value=2 ** 70),
                     st.floats(allow_nan=True, allow_infinity=True), st.text(max_size=12), st.binary(max_size=4))
_keys = st.one_of(st.text(max_size=6), st.integers(min_value=-2 ** 65, max_value=2 ** 65), st.floats(), st.none(), st.booleans(),
                  st.binary(max_size=3))
_values = st.recursive(_scalars, lambda kids: st.one_of(st.lists(kids, max_size=5), st.tuples(kids, kids),
                                                      st.dictionaries(_keys, kids, max_size=5)), max_leaves=30)


@settings(max_examples=600, deadline=None)
@given(_values)
def test_function_hypothesis(lib, v):
    check_function(lib, frame_one(v), "identity")


# ---------------------------------------------------------------------------------------------- 3. endpoint: T(E)
def endpoint_records():
    from tests.golden.make_ref_endpoint_golden import bodies
    out = []
    for h in HANDLERS:
        for b in bodies():
            outcome, e = EP.run_endpoint_request(b, h)
            if outcome == EP.OK:
                out.append(e)
    for v in plain_values():
        try:
            out.append(EP.render(v))
        except (TypeError, ValueError, RecursionError):
            pass
    return out


def test_endpoint_records_equal_json_dumps(lib):
    """The endpoint corpus's response bodies E (all four handlers) and plain values rendered by JSONResponse: T(E) is
    json.dumps of the result, and the oracle's endpoint_text is the same transform."""
    recs = endpoint_records()
    assert len(recs) > 500
    for e in recs:
        want = json.dumps(json.loads(e)).encode()
        assert device_endpoint(lib, e) == want, e
        assert cb.endpoint_text(e) == want, e
        assert cb.endpoint_callback("COMPLETE", e) == (cb.CB_POST, want)


@settings(max_examples=600, deadline=None)
@given(st.recursive(st.one_of(st.none(), st.booleans(), st.integers(), st.floats(allow_nan=False, allow_infinity=False), st.text()),
                    lambda kids: st.one_of(st.lists(kids, max_size=5), st.dictionaries(st.text(max_size=6), kids, max_size=5)),
                    max_leaves=30))
def test_endpoint_hypothesis(lib, v):
    e = EP.render(v)
    assert device_endpoint(lib, e) == json.dumps(v).encode()


def test_endpoint_mutations(lib):
    """30,000 single-byte mutations of endpoint records (malformed UTF-8, stray quotes and backslashes): the device's
    transform is the oracle's, byte for byte."""
    recs = [e for e in endpoint_records() if e]
    rng = random.Random(17)
    for _ in range(30000):
        e = bytearray(rng.choice(recs))
        i = rng.randrange(len(e))
        e[i] = rng.choice([rng.randrange(256), 0x22, 0x5C, 0x2C, 0x3A, 0x7F, 0x80, 0xC3, 0xED, 0xF0, 0xFF])
        e = bytes(e)
        assert device_endpoint(lib, e) == cb.endpoint_text(e), e


# ---------------------------------------------------------------------------------------------- 4. the rules vs the reference
def _golden():
    return json.load(open(os.path.join(HERE, "golden", "ref_callback_runners_golden.json")))


def _safe_kwargs(blob):
    try:
        kw = funcloop.load_args(blob).get("kwargs") or {}
    except Exception:
        return {}
    return kw if isinstance(kw, dict) else {}


def _postable(url):
    import requests
    try:
        requests.Request("POST", url).prepare()
    except requests.exceptions.RequestException:
        return False
    return True


@pytest.mark.parametrize("handler", HANDLERS)
def test_function_rules_equal_the_reference_runner(handler):
    """Per blob, the reference function runner's own callback (ref_callback_runners_golden.json) against the restatement:
    the status; for B9_CB_POST exactly one signed body, {"data": D}, posted as signed to the task's URL or the stub's;
    for B9_CB_UNSENDABLE either nothing signed (json.dumps raised, and the exception escaped the runner's retries) or a
    signed body that requests refused; ERROR signs its own body, which the host builds."""
    from tests.golden.make_ref_callback_runners_golden import STUB_URL, body_digest, function_blobs
    g = _golden()
    blobs = function_blobs()
    rows = g["function"]["handlers"][handler]
    assert len(rows) == len(blobs) == g["function"]["n"]
    kinds = set()
    for blob, row in zip(blobs, rows):
        status, res = funcloop.run_function_task(blob, handler)
        assert row["status"] == status, (blob, row)
        kind, d, url = cb.function_callback(status, cloudpickle.loads(res) if status == "COMPLETE" else None, _safe_kwargs(blob))
        kinds.add(kind)
        if kind == cb.CB_POST:
            # requests refuses a URL without a scheme ("u") before sending: signed, then not posted; the gateway's client
            # meets the same URL
            assert row["signed"] == [body_digest(cb0.BODY_PREFIX + d + b"}")] and row["posted"] == ("=" if _postable(url or STUB_URL) else "-"), (blob, row)
            assert row["url"] == (url or STUB_URL) and row["raised"] is None, (blob, row)
        elif kind == cb.CB_UNSENDABLE:
            assert (row["signed"] == [] and row["raised"] == "TypeError") or (len(row["signed"]) == 1 and row["posted"] == "R"), (blob, row)
        elif status == "ERROR":
            assert row["signed"] == 1, (blob, row)
    assert cb.CB_POST in kinds and (handler != "identity" or cb.CB_UNSENDABLE in kinds)


@pytest.mark.parametrize("handler", HANDLERS)
def test_endpoint_rules_equal_the_reference_runner(handler):
    """Per body, the reference endpoint runner (middleware.run_task around the manager's route) against the restatement:
    a body the gateway refuses has no task (B9_CB_NONE); every answered request signs {"data": D} with D = T(E), falsy
    results included, posted as signed to the stub's URL; a handler that raised is ERROR (the host's traceback body); a
    result JSONResponse cannot render stays COMPLETE and is refused by requests (left to the host on the device)."""
    from tests.golden.make_ref_callback_runners_golden import STUB_URL, body_digest, endpoint_bodies
    g = _golden()
    bodies = endpoint_bodies()
    rows = g["endpoint"]["handlers"][handler]
    assert len(rows) == len(bodies) == g["endpoint"]["n"]
    for b, row in zip(bodies, rows):
        outcome, e = EP.run_endpoint_request(b, handler)
        if outcome == EP.BAD_REQUEST:
            assert row is None and cb.endpoint_callback("REJECTED", None)[0] == cb.CB_NONE
        elif outcome == EP.OK:
            kind, d = cb.endpoint_callback("COMPLETE", e)
            assert kind == cb.CB_POST and row["status"] == "COMPLETE", (b, row)
            assert row["signed"] == [body_digest(cb0.BODY_PREFIX + d + b"}")] and row["posted"] == "=" and row["url"] == STUB_URL, (b, row)
        elif outcome == EP.HANDLER_RAISED:
            assert row["status"] == "ERROR" and row["signed"] == 1 and cb.endpoint_callback("ERROR", None)[0] == cb.CB_HOST, (b, row)
        else:
            assert outcome == EP.RENDER_FAILED and row["status"] == "COMPLETE" and row["posted"] == "R", (b, row)
