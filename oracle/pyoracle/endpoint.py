"""CPU ORACLE (test infrastructure): one request to a non-ASGI `@endpoint`, end to end.

Restates, strictly in the reference's order:

  gateway   pkg/abstractions/endpoint/buffer.go:460-508     SerializeHttpPayload(body); on error 400
                                                             {"error":"invalid request payload"}; otherwise
                                                             json.Marshal(TaskPayload) to the container
                                                             (pkg/types/task.go:13-16: nil Args -> "args":null)
  runner    sdk/src/beta9/runner/endpoint.py:202-306         payload = json.loads(body); args / kwargs None -> [] / {};
                                                             handler(*args, **kwargs); a raise -> 500
  response  endpoint.py:256-267                              JSONResponse(result).body; a render failure -> 500
                                                             with the task Complete

JSONResponse.render is json.dumps(ensure_ascii=False, allow_nan=False, indent=None, separators=(",", ":")) encoded as
UTF-8 (Starlette). PINNED by tests/golden/ref_endpoint_golden.json, which the reference's own EndpointManager produced
(tests/golden/make_ref_endpoint_golden.py); the Go halves are the restatements in httpserialize.py / gojson.py.
"""
from __future__ import annotations

import json
from typing import Any, Callable, Optional, Tuple, Union

from .gojson import go_marshal
from .handlers import HANDLERS
from .httpserialize import InvalidRequestPayload, serialize_http_payload

OK = 200
BAD_REQUEST = 400
HANDLER_RAISED = "500-handler"
RENDER_FAILED = "500-render"
INVALID_PAYLOAD_BODY = b'{"error":"invalid request payload"}'


def render(result: Any) -> bytes:
    """Starlette JSONResponse(result).body."""
    return json.dumps(result, ensure_ascii=False, allow_nan=False, indent=None, separators=(",", ":")).encode("utf-8")


def gateway_body(body: bytes) -> bytes:
    """What the gateway forwards to the container: json.Marshal(TaskPayload{Args, Kwargs}). Raises
    InvalidRequestPayload where it answers 400."""
    args, kwargs = serialize_http_payload(body)
    return ('{"args":' + go_marshal(args) + ',"kwargs":' + go_marshal(kwargs) + "}").encode("utf-8")


def run_endpoint_request(body: bytes, handler: Union[str, Callable[..., Any]]) -> Tuple[Union[int, str], Optional[bytes]]:
    """-> (outcome, bytes): (200, response body), (400, the gateway's body), ("500-handler", None) when the handler
    raised, ("500-render", None) when JSONResponse could not render the result."""
    fn = HANDLERS[handler] if isinstance(handler, str) else handler
    try:
        forwarded = gateway_body(body)
    except InvalidRequestPayload:
        return BAD_REQUEST, INVALID_PAYLOAD_BODY
    payload = json.loads(forwarded)
    args = payload.get("args", [])
    if args is None:
        args = []
    kwargs = payload.get("kwargs", {})
    if kwargs is None:
        kwargs = {}
    try:
        result = fn(*args, **kwargs)
    except BaseException:
        return HANDLER_RAISED, None
    try:
        return OK, render(result)
    except BaseException:
        return RENDER_FAILED, None
