"""Task callbacks on a CPU: the oracle's restatement of send_callback against the reference runner's own callbacks
(tests/golden/ref_callback_golden.json), and the device's signing code (beta9_b200/csrc/callback_sign.cuh, built for the
host through tests/host_shim/callback_shim.cpp) against hashlib / hmac / base64 and json."""
import base64
import ctypes as C
import hashlib
import hmac
import json
import os
import subprocess
import uuid

import pytest

from oracle.pyoracle import callback as cb
from oracle.pyoracle.handlers import HANDLERS as FUNCS
from tests.golden.make_ref_callback_golden import KEY, STUB_URL, TS, explicit_wires, headers_digest, signed_digest, url_letter
from tests.golden.make_ref_retry_golden import corpus_wires
from tests.golden.make_ref_runner_golden import HANDLERS
from tests.retry_oracle import call_handler

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_shim", "callback_shim.cpp")
SO = os.path.join(HERE, "host_shim", "libcallback.so")
GXX = os.environ.get("CXX", "g++")


def _golden():
    return json.load(open(os.path.join(HERE, "golden", "ref_callback_golden.json")))


# ---------------------------------------------------------------------------------------------- 1. the oracle vs the runner
@pytest.mark.parametrize("handler", HANDLERS)
def test_oracle_callback_equals_the_reference_runner(handler):
    """Per task: the status, that the runner signs {"data": ...} built from the record (every signed body, in order, under
    one hash), that requests posts those bytes or refuses them exactly where the oracle's kind says so, the URL (the
    stub's, or a callback_url override) and the X-Task-ID / X-Task-Status headers."""
    g = _golden()
    assert (g["stub_url"], g["key"].encode(), g["ts"]) == (STUB_URL, KEY, TS)
    ref = g["handlers"][handler]
    wires = corpus_wires(handler) + explicit_wires(handler)
    assert len(wires) == ref["n"] and len(wires) > 1000
    status_l, posted_l, url_l, bodies, hdrs, kinds = "", "", "", [], [], set()
    for w in wires:
        t = json.loads(w)
        tid = uuid.UUID(t["task_id"]).bytes
        status, result, _ = call_handler(FUNCS[handler], t["args"], t["kwargs"], ())
        kind = cb.callback_kind(status, result, t["kwargs"])
        kinds.add(kind)
        body = cb.callback_body(result)
        status_l += {"COMPLETE": "C", "ERROR": "E"}[status]
        bodies.append(body)                                  # the runner signs every completed task's body
        want = cb.runner_callback(tid, status, result, t["kwargs"], STUB_URL, KEY, TS)
        url = (t["kwargs"] or {}).get("callback_url") or STUB_URL
        if kind == cb.CB_UNSENDABLE:
            assert want is None
            posted_l += "R"
        elif isinstance(url, str):
            assert want is not None and want[:2] == (url, body)
            assert want[2] == cb.callback_headers(tid, status, cb.sign_payload(body, KEY, TS)[0], TS)
            posted_l += "="
        else:
            assert kind == cb.CB_HOST              # a URL requests cannot use: the runner's post raises, and is caught
            posted_l += "-"
        url_l += url_letter(url)
        hdrs.append((str(uuid.UUID(bytes=tid)), status))
        if kind == cb.CB_HOST:
            assert "callback_url" in t["kwargs"]
    assert ref["status"] == status_l
    assert ref["signed"] == "S" * len(wires)
    assert ref["posted"] == posted_l
    assert ref["url"] == url_l
    assert ref["signed_sha256"] == signed_digest(bodies)
    assert ref["headers_sha256"] == headers_digest(hdrs)
    for row, w in zip(ref["explicit"], wires[-len(ref["explicit"]):]):
        t = json.loads(w)
        _, result, _ = call_handler(FUNCS[handler], t["args"], t["kwargs"], ())
        assert row[1].encode() == cb.callback_body(result)
    assert cb.CB_POST in kinds


def test_oracle_kinds_of_the_statuses_the_runner_never_calls_back():
    assert cb.callback_kind("RETRY", None) == cb.callback_kind("RETRY_LIMIT", None) == cb.callback_kind("REJECTED", None) == cb.CB_NONE
    assert cb.callback_kind("UNSUPPORTED", None) == cb.callback_kind("COMPLETE", b'"x"', pickle=True) == cb.CB_HOST
    for r in (b"NaN", b"Infinity", b"-Infinity"):
        assert cb.callback_kind("COMPLETE", r) == cb.CB_UNSENDABLE
    assert cb.callback_kind("ERROR", None, {"callback_url": None}) == cb.CB_HOST
    assert cb.sign_payload(cb.EMPTY_BODY, b"", 123) == ("", 0)
    assert base64.b64encode(cb.BODY_PREFIX) == b"eyJkYXRhIjog"


# ---------------------------------------------------------------------------------------------- 2. the device's code
@pytest.fixture(scope="module")
def dev():
    csrc = os.path.join(os.path.dirname(HERE), "beta9_b200", "csrc")
    deps = [os.path.join(csrc, f) for f in ("callback_sign.cuh", "json_device.cuh")]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max([os.path.getmtime(SRC)] + [os.path.getmtime(d) for d in deps]):
        r = subprocess.run([GXX, "-O2", "-std=c++17", "-shared", "-fPIC", "-o", SO, SRC], capture_output=True, text=True)
        if r.returncode:
            pytest.skip("no host C++ compiler for the shim: " + r.stderr[-300:])
    lib = C.CDLL(SO)
    lib.b9_cb_sha256.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p]
    lib.b9_cb_hmac.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint64, C.c_void_p]
    lib.b9_cb_sign_record.argtypes = [C.c_char_p, C.c_uint32, C.c_int64, C.c_char_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32)]
    lib.b9_cb_nonfinite.argtypes = [C.c_char_p, C.c_uint32]
    lib.b9_cb_kwargs_have_callback_url.argtypes = [C.c_char_p, C.c_uint32, C.c_int]
    return lib


def _sha(lib, m: bytes) -> bytes:
    o = (C.c_uint8 * 32)()
    lib.b9_cb_sha256(m, len(m), o)
    return bytes(o)


def _hmac(lib, key: bytes, m: bytes) -> bytes:
    o = (C.c_uint8 * 32)()
    lib.b9_cb_hmac(key, len(key), m, len(m), o)
    return bytes(o)


def _record(lib, key: bytes, ts: int, r: bytes):
    o = (C.c_uint8 * 32)()
    blocks = C.c_uint32(0)
    lib.b9_cb_sign_record(key, len(key), ts, r, len(r), o, C.byref(blocks))
    return bytes(o), int(blocks.value)


def test_sha256_nist_vectors(dev):
    # FIPS 180-2 appendix B
    assert _sha(dev, b"abc").hex() == "ba7816bf8f01cfea414140de5dae2223b00361a396177a9cb410ff61f20015ad"
    assert _sha(dev, b"abcdbcdecdefdefgefghfghighijhijkijkljklmklmnlmnomnopnopq").hex() == \
        "248d6a61d20638b8e5c026930c3e6039a33ce45964ff2167f6ecedd419db06c1"
    assert _sha(dev, b"a" * 1000000).hex() == "cdc76e5c9914fb9281a1c7e284d73e67f1809a48a497200e046d39ccc7112cd0"
    assert _sha(dev, b"").hex() == "e3b0c44298fc1c149afbf4c8996fb92427ae41e4649b934ca495991b7852b855"


def test_sha256_every_length_to_4096(dev):
    m = bytes((i * 131 + 7) & 0xFF for i in range(4097))
    for n in range(4097):
        assert _sha(dev, m[:n]) == hashlib.sha256(m[:n]).digest(), n


RFC4231 = [   # (key, data, HMAC-SHA256), RFC 4231 test cases 1-4, 6, 7
    (b"\x0b" * 20, b"Hi There", "b0344c61d8db38535ca8afceaf0bf12b881dc200c9833da726e9376c2e32cff7"),
    (b"Jefe", b"what do ya want for nothing?", "5bdcc146bf60754e6a042426089575c75a003f089d2739839dec58b964ec3843"),
    (b"\xaa" * 20, b"\xdd" * 50, "773ea91e36800e46854db8ebd09181a72959098b3ef8c122d9635514ced565fe"),
    (bytes(range(1, 26)), b"\xcd" * 50, "82558a389a443c0ea4cc819899f2083a85f0faa3e578f8077a2e3ff46729665b"),
    (b"\xaa" * 131, b"Test Using Larger Than Block-Size Key - Hash Key First",
     "60e431591ee0b67f0d8a26aacbf5b77f8e0bc6213728c5140546040f0ee37f54"),
    (b"\xaa" * 131, b"This is a test using a larger than block-size key and a larger than block-size data. The key needs to be "
                    b"hashed before being used by the HMAC algorithm.",
     "9b09ffa71b942fcb27635fbcd5b0e944bfdc63644f0713938a7f51535c3a35e2"),
]


def test_hmac_rfc4231_vectors(dev):
    for key, data, want in RFC4231:
        assert _hmac(dev, key, data).hex() == want


@pytest.mark.parametrize("key_len", [0, 1, 63, 64, 65, 200])
def test_hmac_key_lengths(dev, key_len):
    key = bytes((i * 29 + 3) & 0xFF for i in range(key_len))
    for n in (0, 1, 55, 56, 63, 64, 65, 119, 120, 1000):
        m = bytes((i * 17) & 0xFF for i in range(n))
        assert _hmac(dev, key, m) == hmac.new(key, m, hashlib.sha256).digest(), (key_len, n)


def _want(key: bytes, ts: int, r: bytes) -> bytes:
    return hmac.new(key, cb.sign_message(cb.callback_body(r), ts), hashlib.sha256).digest()


def _blocks(r: bytes, ts: int) -> int:
    """Inner compressions of one record (the issue's count): ceil((12 + 4 ceil((len R + 1) / 3) + 1 + digits + 9) / 64)."""
    return -(-(12 + 4 * -(-(len(r) + 1) // 3) + 1 + len(str(ts)) + 9) // 64)


@pytest.mark.parametrize("ts", [0, 9, 10, 10**9, 2**63 - 1])
def test_record_signature_timestamps(dev, ts):
    key = b"k" * 32
    for r in (b"", b"{}", b'"x"', b"12345", b"[1, 2, 3]", bytes(range(256)) * 3):
        d, blocks = _record(dev, key, ts, r)
        assert d == _want(key, ts, r), (ts, r[:20])
        assert blocks == _blocks(r, ts)


def test_record_signature_every_length_and_residue(dev):
    """Every result length 0-4096 covers every len mod 3 (the base64 tail: '==', '=' or none); timestamps of 1 to 19
    digits over the first 64 lengths put the signed message at every residue mod 64, 55 / 56 / 63 / 0 (the pad byte
    and the length words at a block's end) included."""
    key = b"workspace-key"
    base = bytes((i * 37 + 11) & 0xFF for i in range(4097))
    for n in range(4097):
        r = base[:n]
        assert _record(dev, key, 1760000000, r)[0] == _want(key, 1760000000, r), n
    residues = set()
    for digits in range(1, 20):
        ts = 10 ** (digits - 1) + 7 if digits > 1 else 7
        for n in range(64):
            r = base[:n]
            assert _record(dev, key, ts, r)[0] == _want(key, ts, r), (ts, n)
            residues.add(len(cb.sign_message(cb.callback_body(r), ts)) % 64)
    assert residues == set(range(64))


@pytest.mark.parametrize("key_len", [0, 1, 63, 64, 65, 200])
def test_record_signature_key_lengths(dev, key_len):
    key = bytes((i * 7 + 1) & 0xFF for i in range(key_len))
    for r in (b"{}", b'"hello"', b"x" * 1000):
        assert _record(dev, key, 1760000000, r)[0] == _want(key, 1760000000, r)


def test_nonfinite(dev):
    for r, want in [(b"NaN", 1), (b"Infinity", 1), (b"-Infinity", 1), (b"1e308", 0), (b'"NaN"', 0), (b"-NaN", 0),
                    (b"Infinity1", 0), (b"", 0), (b"inf", 0)]:
        assert dev.b9_cb_nonfinite(r, len(r)) == want, r


KW_CASES = [   # (payload, mode, has a "callback_url" kwarg as the runner sees it)
    (b'{"args": ["x"], "kwargs": {"callback_url": "u"}}', 0, True),
    (b'{"args": ["x"], "kwargs": {"callback_url": null}}', 0, True),
    (b'{"args": ["x"], "kwargs": {"a": 1, "callback_url": 1}}', 0, True),
    (b'{"args": ["x"], "kwargs": {"callback\\u005furl": ""}}', 0, True),
    (b'{"args": ["x"], "KWARGS": {"callback_url": ""}}', 0, True),             # struct keys fold case
    (b'{"args": ["x"], "kwargs": {"callback_url": 1}, "kwargs": {"b": 2}}', 0, True),   # maps merge
    (b'{"args": ["x"], "kwargs": {"callback_url": 1}, "kwargs": null, "kwargs": {"b": 2}}', 0, False),   # null resets
    (b'{"args": ["callback_url"], "kwargs": {"Callback_url": 1}}', 0, False),
    (b'{"args": ["x"], "kwargs": {"k": {"callback_url": 1}}}', 0, False),
    (b'{"args": ["x"], "kwargs": {}}', 0, False),
    (b'{"args": ["x"], "callback_url": "u"}', 0, False),
    (b'{"args": ["x"], "callback_url": "u"}', 1, True),                        # an HTTP body's other keys are kwargs
    (b'{"args": ["x"], "kwargs": {"a": 1}, "callback_url": "u"}', 1, False),
    (b'{"args": ["x"], "kwargs": {"callback_url": 1}}', 1, True),
    (b'{"args": ["x"], "kwargs": 5, "callback_url": "u"}', 1, True),
    (b'{"args": ["x"], "KWARGS": {"callback_url": 1}}', 1, False),             # map keys are exact: "KWARGS" is a kwarg
    (b'{"task_id": "t", "args": ["x"], "kwargs": {"callback_url": "u"}}', 2, True),
    (b'{"task_id": "t", "args": ["x"], "kwargs": null}', 2, False),
    (b'{"task_id": "t", "args": ["x"], "kwargs": {"z": 1}}', 2, False),
]


def test_kwargs_callback_url(dev):
    for p, mode, want in KW_CASES:
        assert dev.b9_cb_kwargs_have_callback_url(p, len(p), mode) == int(want), (p, mode)
