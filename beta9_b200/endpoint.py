"""Host-side mirror of the reference's `@endpoint` surface for request/response traffic: each HTTP request body becomes
one task, answered by the device with the bytes the endpoint's runner would send.

  Endpoint / _CallableWrapper   sdk/src/beta9/abstractions/endpoint.py (the decorator; resource arguments kept for
                                API compatibility)
  gateway                       pkg/abstractions/endpoint/buffer.go:460-572 (SerializeHttpPayload: a body it refuses is
                                400 {"error":"invalid request payload"}; the container's status and body are copied back)
  runner                        sdk/src/beta9/runner/endpoint.py:202-306 (handler(*args, **kwargs) -> JSONResponse)

Requests go in one at a time through b9_submit with B9_TF_HTTP_BODY (the gateway's RequestBuffer pattern: any thread,
micro-batched by the library), then b9_flush and endpoint drains (b9_endpoint_drain_launch). Each request returns
(http_status, body | None): 200 with the response bytes, 400 with the gateway's body, 500 with None (the handler raised;
the runner's body is its traceback text, which only a Python runner can compose). There is no CPU fallback in this
package: a request the device does not answer (B9_ST_UNSUPPORTED, include/b9gpu.h) is listed in `.unsupported` and
returns (None, None), for the host to route through the reference's path.
"""
from __future__ import annotations

import os
import uuid
from typing import Any, Callable, List, Optional, Sequence, Tuple

from . import _lib as L
from .device_queue import DeviceQueue

ENDPOINT_STUB_TYPE = "endpoint"
INVALID_PAYLOAD_BODY = b'{"error":"invalid request payload"}'      # buffer.go:465-477


class Endpoint:
    """Decorator; resource arguments are kept for API compatibility."""

    def __init__(self, cpu: Any = 1.0, memory: Any = 128, gpu: Any = "", image: Any = None, timeout: int = 180, workers: int = 1,
                 name: Optional[str] = None, gpu_handler: Optional[str] = None, device: int = 0,
                 queue: Optional[DeviceQueue] = None, callback_url: Optional[str] = None, signing_key: Optional[bytes] = None,
                 **kwargs: Any):
        self.cpu, self.memory, self.gpu, self.image, self.timeout, self.workers = cpu, memory, gpu, image, timeout, workers
        self.name = name
        self.gpu_handler = gpu_handler or os.environ.get("B9_GPU_HANDLER", "identity")
        self.device = device
        # the stub's callback URL: the device settles and signs the runner's callback of every answered request
        # (b9_set_callback_runners), with the workspace's signing_key (None or b"": unsigned); nothing is posted here
        self.callback_url = callback_url
        self.signing_key = bytes(signing_key or b"")
        self._cb_set = False
        self.extra = kwargs
        self._queue = queue
        self.stub_id = str(uuid.uuid4())

    @property
    def queue(self) -> DeviceQueue:
        if self._queue is None:
            self._queue = DeviceQueue(device=self.device)     # raises without a GPU: no CPU path
        return self._queue

    def __call__(self, func: Callable) -> "_CallableWrapper":
        return _CallableWrapper(func, self)


class _CallableWrapper:
    base_stub_type = ENDPOINT_STUB_TYPE

    def __init__(self, func: Callable, parent: Endpoint):
        self.func = func
        self.parent = parent
        self.unsupported: List[bytes] = []        # request bodies the device did not answer (status UNSUPPORTED)
        # with a callback_url: per body of the last call, what the runner hands requests.post, (url, body bytes, headers),
        # or None (no task: a 400; or a callback left to the host, such as an ERROR's traceback)
        self.callbacks: List[Optional[tuple]] = []

    def local(self, *args: Any, **kwargs: Any) -> Any:
        return self.func(*args, **kwargs)

    def __call__(self, *args: Any, **kwargs: Any) -> Any:
        return self.local(*args, **kwargs)

    def request(self, body: bytes) -> Tuple[Optional[int], Optional[bytes]]:
        """One HTTP request body -> (http_status, response body | None)."""
        return self.requests([body])[0]

    def requests(self, bodies: Sequence[bytes]) -> List[Tuple[Optional[int], Optional[bytes]]]:
        """Many request bodies -> one (http_status, response body | None) per body, in input order."""
        q = self.parent.queue
        bodies = [bytes(b) for b in bodies]
        ids = [uuid.uuid4().bytes for _ in bodies]
        for tid, b in zip(ids, bodies):
            q.submit(tid, b, L.TF_HTTP_BODY)
        q.flush()
        want = {tid: k for k, tid in enumerate(ids)}
        out: List[Optional[Tuple[Optional[int], Optional[bytes]]]] = [None] * len(bodies)
        cb = bool(self.parent.callback_url)
        if cb and not self.parent._cb_set:
            q.set_callback_policy(self.parent.signing_key)
            q.set_callback_runners(endpoint=True)
            self.parent._cb_set = True
        self.callbacks = [None] * len(bodies)
        seen = 0
        while seen < len(bodies):
            r = q.drain(self.parent.gpu_handler, endpoint=True, callbacks=cb)
            if r.n == 0:
                break
            for i in range(r.n):
                k = want.get(r.task_ids[i].tobytes())
                if k is None:
                    continue
                st = int(r.status[i])
                if cb and int(r.cb_kind[i]) == L.CB_POST:
                    self.callbacks[k] = (self.parent.callback_url, r.callback_body(i), r.callback_headers(i))
                if st == L.ST_COMPLETE:
                    out[k] = (200, r.result(i))
                elif st == L.ST_REJECTED:
                    out[k] = (400, INVALID_PAYLOAD_BODY)
                elif st == L.ST_ERROR:
                    out[k] = (500, None)
                else:
                    self.unsupported.append(bodies[k])
                    out[k] = (None, None)
                seen += 1
        if seen < len(bodies):
            raise L.B9Error(L.B9_EIO, f"{len(bodies) - seen} of {len(bodies)} requests did not come back from the queue")
        return out  # type: ignore[return-value]


def endpoint(*args: Any, **kwargs: Any) -> Endpoint:
    """`@endpoint(...)` spelling of the decorator."""
    return Endpoint(*args, **kwargs)
