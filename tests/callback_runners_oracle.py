"""The function and endpoint runners' callbacks, restated (the task-queue runner's is oracle/pyoracle/callback.py): which
request send_callback sends after a function or endpoint task, and the JSON D it signs and posts as {"data": D}.

    runner/common.py:406-481      url = override_callback_url or context.callback_url; body = {"data": payload};
                                  sign_payload(json.dumps(body)); requests.post(url, json=body) (allow_nan=False)
    runner/function.py:235-343    payload = the handler's result (not `result or {}`); callback_url = kwargs.pop(...)
    middleware.py:29-78           payload = the endpoint handler's result, whose JSONResponse body is the drain's record
"""
from __future__ import annotations

import json
from typing import Any, Dict, Optional, Tuple

from oracle.pyoracle.callback import CB_HOST, CB_NONE, CB_POST, CB_UNSENDABLE  # noqa: F401


# Both end in send_callback too (runner/common.py:406-481), with payload = the handler's result itself (no `or {}`): the
# body is json.dumps({"data": result}) with the defaults, i.e. BODY_PREFIX + D + b"}" for D = json.dumps(result).
MAX_BODY = 1 << 20           # a D longer than this is left to the host (callback_runners.cuh, CBR_MAX_BODY)
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1


def _scan(v: Any, found: Dict[str, bool]) -> None:
    """What json.dumps / requests make of a plain value: bytes (TypeError), a non-finite float (requests' allow_nan=False),
    an int outside int64 (which the device does not write); dict keys included."""
    if isinstance(v, (bytes, bytearray)):
        found["bytes"] = True
    elif isinstance(v, bool) or v is None or isinstance(v, str):
        pass
    elif isinstance(v, int):
        found["host"] |= not (INT64_MIN <= v <= INT64_MAX)
    elif isinstance(v, float):
        found["nonfinite"] |= v != v or v in (float("inf"), float("-inf"))
    elif isinstance(v, (list, tuple)):
        for x in v:
            _scan(x, found)
    elif isinstance(v, dict):
        for k, x in v.items():
            _scan(k, found)
            _scan(x, found)
    else:
        found["host"] = True


def function_callback(status: str, result: Any, kwargs: Optional[Dict[str, Any]]) -> Tuple[int, Optional[bytes], Optional[str]]:
    """The function runner's callback for one pickle record (runner/function.py:235-343) under B9_CB_RUNNER_FUNCTION:
    (kind, D, url) with D = json.dumps(result) for B9_CB_POST (else None), url = the task's callback_url kwarg when it is a
    truthy str the device posts to, None for the stub's. status: the record's; result: the handler's return value.
    Precedence: a non-str callback_url first (HOST), then bytes or a non-finite float anywhere (UNSENDABLE), then an int
    outside int64 or a D past MAX_BODY (HOST). The device walks the value in json.dumps order and stops once D passes
    MAX_BODY, so for a value whose bytes or non-finite float come only after that point it answers HOST where this
    answers UNSENDABLE (HOST is always safe: the host settles the record); no test value is that large."""
    if status != "COMPLETE":
        return CB_HOST, None, None                  # ERROR's body holds the exception text; UNSUPPORTED is the host's
    url = (kwargs or {}).get("callback_url")
    if url:
        if not isinstance(url, str):
            return CB_HOST, None, None
        try:
            url.encode("utf-8")
        except UnicodeEncodeError:                  # a lone surrogate: not bytes the device hands over
            return CB_HOST, None, None
    else:
        url = None
    found = {"bytes": False, "nonfinite": False, "host": False}
    _scan(result, found)
    if found["bytes"] or found["nonfinite"]:
        return CB_UNSENDABLE, None, None            # json.dumps raises, or requests refuses the signed body
    if found["host"]:
        return CB_HOST, None, None
    d = json.dumps(result).encode()
    if len(d) > MAX_BODY:
        return CB_HOST, None, None
    return CB_POST, d, url


def endpoint_text(e: bytes) -> bytes:
    """T(E): the endpoint record's compact ensure_ascii=False JSON re-spaced (", " / ": " outside strings) and with every
    code point from U+0080 and the byte 0x7F inside strings as \\uXXXX (a pair above U+FFFF); E's own escapes as they are.
    A malformed UTF-8 byte (a corrupted record) becomes \\u00XX. For E = JSONResponse(x).body this is json.dumps(x)."""
    out = bytearray()

    def u(cp: int) -> None:
        if cp >= 0x10000:
            v = cp - 0x10000
            out.extend(b"\\u%04x\\u%04x" % (0xD800 + (v >> 10), 0xDC00 + (v & 0x3FF)))
        else:
            out.extend(b"\\u%04x" % cp)

    def seq(i: int) -> int:
        c = e[i]
        n = 2 if 0xC2 <= c <= 0xDF else 3 if 0xE0 <= c <= 0xEF else 4 if 0xF0 <= c <= 0xF4 else 0
        if not n or i + n > len(e):
            return 0
        lo = {0xE0: 0xA0, 0xF0: 0x90}.get(c, 0x80)
        hi = 0x8F if c == 0xF4 else 0xBF
        if not lo <= e[i + 1] <= hi or any(not 0x80 <= e[i + k] <= 0xBF for k in range(2, n)):
            return 0
        return n

    in_str, i = False, 0
    while i < len(e):
        c = e[i]
        if not in_str:
            out.append(c)
            if c == 0x22:
                in_str = True
            elif c in (0x2C, 0x3A):
                out.append(0x20)
            i += 1
        elif c == 0x5C:
            out.extend(e[i:i + 2])
            i += 2
        elif c == 0x22:
            out.append(c)
            in_str = False
            i += 1
        elif c < 0x7F:
            out.append(c)
            i += 1
        else:
            n = seq(i) if c >= 0x80 else 0
            if n:
                u(ord(e[i:i + n].decode("utf-8", "surrogatepass")))
                i += n
            else:
                u(c)
                i += 1
    return bytes(out)


def endpoint_callback(status: str, record: Optional[bytes]) -> Tuple[int, Optional[bytes]]:
    """The endpoint runner's callback for one record of an endpoint drain (middleware.py:29-78) under
    B9_CB_RUNNER_ENDPOINT: (kind, D). COMPLETE posts json.dumps(result) = T(E); REJECTED is the gateway's 400 (no task);
    ERROR's body is the traceback and UNSUPPORTED is the host's."""
    if status == "REJECTED":
        return CB_NONE, None
    if status != "COMPLETE" or record is None:
        return CB_HOST, None
    d = endpoint_text(record)
    if len(d) > MAX_BODY:
        return CB_HOST, None
    return CB_POST, d
