"""The task callback of the task-queue runner, restated: which request `send_callback` sends after a task, its body, its
headers, and the gateway's signature over it.

    runner/taskqueue.py:391-397   after task_queue_complete (not for Retry: `continue`):
                                  send_callback(payload=result or {}, task_status, override_callback_url=kwargs.get("callback_url"))
    runner/common.py:430-481      url = override or context.callback_url; body = {"data": payload};
                                  sign_payload(json.dumps(body).encode()); requests.post(url, json=body, headers=...)
    pkg/auth/sign.go:17-35        hex(HMAC-SHA256(key, base64.StdEncoding(payload) + ":" + Unix seconds))

The body the runner signs is json.dumps(body); the body requests posts is complexjson.dumps(body, allow_nan=False): the
same bytes, or InvalidJSONError for a non-finite float (then nothing is posted). For a result whose serialize_result
bytes are R, both are b'{"data": ' + R + b'}'. The Go half (SignPayload) is a restatement here, unpinned by a golden.
"""
from __future__ import annotations

import base64
import hashlib
import hmac
import json
import uuid
from typing import Any, Dict, Optional, Tuple

# enum b9_callback_kind (include/b9gpu.h)
CB_NONE, CB_POST, CB_UNSENDABLE, CB_HOST = 0, 1, 2, 3
KIND_NAMES = {CB_NONE: "NONE", CB_POST: "POST", CB_UNSENDABLE: "UNSENDABLE", CB_HOST: "HOST"}
BODY_PREFIX = b'{"data": '
EMPTY_BODY = b'{"data": {}}'


def callback_body(result: Optional[bytes]) -> bytes:
    """The body of a task's callback from its record's result bytes (None: has_result = 0, the runner's `result or {}`)."""
    return BODY_PREFIX + (result if result is not None else b"{}") + b"}"


def sign_payload(payload: bytes, key: bytes, ts: int) -> Tuple[str, int]:
    """SignPayload (pkg/auth/sign.go:17-35) at Unix time `ts`. An empty key is the gateway's Ok: false answer
    (services/auth.go:64-83): the runner's headers then carry the response's defaults, "" and 0."""
    if not key:
        return "", 0
    msg = base64.b64encode(payload) + b":%d" % ts
    return hmac.new(key, msg, hashlib.sha256).hexdigest(), ts


def sign_message(body: bytes, ts: int) -> bytes:
    """The bytes SignPayload hashes for this body."""
    return base64.b64encode(body) + b":%d" % ts


def is_unsendable(result: Optional[bytes]) -> bool:
    """requests refuses the body: the result holds a non-finite float (allow_nan=False)."""
    if result is None:
        return False
    try:
        json.dumps({"data": json.loads(result)}, allow_nan=False)
    except ValueError:
        return True
    return False


def callback_kind(status: str, result: Optional[bytes], kwargs: Optional[Dict[str, Any]] = None, pickle: bool = False) -> int:
    """The device's b9_callback_kind for one task-queue record: status as the runner / the drain reports it, the
    record's result bytes (None without), the kwargs the runner called the handler with."""
    if pickle or status == "UNSUPPORTED":
        return CB_HOST
    if status in ("RETRY", "RETRY_LIMIT", "REJECTED"):
        return CB_NONE
    if status == "ERROR" and kwargs and "callback_url" in kwargs:
        return CB_HOST                          # the runner posts to that value (or to the stub's URL when it is falsy)
    if status == "COMPLETE" and is_unsendable(result):
        return CB_UNSENDABLE
    return CB_POST


def callback_headers(task_id: bytes, status: str, signature: str, ts: int) -> Dict[str, str]:
    """send_callback's headers (runner/common.py:463-469); task_id: 16 raw UUID bytes."""
    return {"X-Task-ID": str(uuid.UUID(bytes=bytes(task_id))), "X-Task-Status": status,
            "X-Task-Signature": signature, "X-Task-Timestamp": str(ts)}


def runner_callback(task_id: bytes, status: str, result: Optional[bytes], kwargs: Optional[Dict[str, Any]],
                    stub_url: Optional[str], key: bytes, ts: int):
    """What the runner hands requests.post for one completed task-queue task: (url, body bytes, headers), or None when it
    posts nothing (Retry, no URL, or a body requests refuses)."""
    if status not in ("COMPLETE", "ERROR"):
        return None
    url = (kwargs or {}).get("callback_url") or stub_url
    if not url:
        return None
    body = callback_body(result)
    sig, t = sign_payload(body, key, ts)
    if status == "COMPLETE" and is_unsendable(result):
        return None
    return url, body, callback_headers(task_id, status, sig, t)
