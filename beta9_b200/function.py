"""Host-side mirror of the reference's `@function` surface for the fan-out path: `.map()` / `.remote()` with the
reference's cloudpickle framing, routed through the batch C ABI instead of one container per input.

  Function / _CallableWrapper   sdk/src/beta9/abstractions/function.py:96-282 (`_call_remote` :198-232, `_format_args`
                                :246-251, `map` :253-282)
  gateway framing rule          pkg/abstractions/function/task.go:84,104-108 (a blob starting 80 05 95 is the runner's
                                argument blob as it is)
  runner loop                   sdk/src/beta9/runner/function.py:236-283 (unpickle -> handler -> cloudpickle.dumps(result))

Every input becomes one task whose payload is exactly the bytes the reference sends (pushed with B9_TF_PICKLE); results
come back as the bytes the reference's runner would have set and are unpickled here like `_call_remote` does. The device
settles the shape the configurations use (one `str` argument, identity), and with `Function(full_pickle=True)` every
handler over plain values (B9_DRAIN_PICKLE_FULL, include/b9gpu.h); other pickles come back UNSUPPORTED — there is no
CPU fallback in this package: their inputs are listed in `.unsupported` for the host to route through the reference loop.
"""
from __future__ import annotations

import os
import uuid
from typing import Any, Callable, Iterator, List, Optional, Sequence, Tuple

import cloudpickle
import numpy as np

from . import _lib as L
from .device_queue import DeviceQueue, STATUS_NAMES

FUNCTION_STUB_TYPE = "function"
TF_PICKLE = 0x04
CLOUDPICKLE_HEADER = b"\x80\x05\x95"


class Function:
    """Decorator; resource arguments are kept for API compatibility (function.py:96-150)."""

    def __init__(self, cpu: Any = 1.0, memory: Any = 128, gpu: Any = "", image: Any = None, timeout: int = 3600, retries: int = 3,
                 name: Optional[str] = None, headless: bool = False, gpu_handler: Optional[str] = None, device: int = 0,
                 queue: Optional[DeviceQueue] = None, full_pickle: bool = False, callback_url: Optional[str] = None,
                 signing_key: Optional[bytes] = None, **kwargs: Any):
        self.cpu, self.memory, self.gpu, self.image, self.timeout, self.retries = cpu, memory, gpu, image, timeout, retries
        self.name, self.headless = name, headless
        self.gpu_handler = gpu_handler or os.environ.get("B9_GPU_HANDLER", "identity")
        self.device = device
        self.full_pickle = full_pickle            # B9_DRAIN_PICKLE_FULL: every handler over plain values, not just one str
        # the stub's callback URL: the device settles and signs the runner's callback of every completed task (full_pickle
        # drains; b9_set_callback_runners), with the workspace's signing_key (None or b"": unsigned); nothing is posted here
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

    def prepare_runtime(self, func: Optional[Callable] = None, stub_type: str = FUNCTION_STUB_TYPE) -> bool:
        return True

    def __call__(self, func: Callable) -> "_CallableWrapper":
        return _CallableWrapper(func, self)


class _CallableWrapper:
    base_stub_type = FUNCTION_STUB_TYPE

    def __init__(self, func: Callable, parent: Function):
        self.func = func
        self.parent = parent
        self.unsupported: List[Any] = []          # inputs whose pickle the device does not settle (status UNSUPPORTED)
        # with a callback_url: per input of the last call, what the runner hands requests.post, (url, body bytes, headers),
        # or None (nothing the device posts: an unsendable body, or a callback left to the host, such as an ERROR's)
        self.callbacks: List[Optional[tuple]] = []

    def __call__(self, *args: Any, **kwargs: Any) -> Any:
        if os.environ.get("CONTAINER_ID") is not None:          # function.py:178-181: inside a container the call is local
            return self.local(*args, **kwargs)
        if not self.parent.prepare_runtime(func=self.func, stub_type=self.base_stub_type):
            return None
        return self._call_remote(*args, **kwargs)

    def local(self, *args: Any, **kwargs: Any) -> Any:
        return self.func(*args, **kwargs)

    def remote(self, *args: Any, **kwargs: Any) -> Any:
        return self(*args, **kwargs)

    @staticmethod
    def _format_args(args: Any) -> List[Any]:
        """function.py:246-251."""
        if isinstance(args, tuple):
            return list(args)
        if not isinstance(args, list):
            return [args]
        return args

    @staticmethod
    def _frame(args: Tuple[Any, ...], kwargs: dict) -> bytes:
        return cloudpickle.dumps({"args": args, "kwargs": kwargs})          # function.py:199-204

    def _run_batch(self, frames: List[bytes]) -> List[Tuple[str, Optional[bytes]]]:
        """One push (B9_TF_PICKLE) + drains until every task is back; -> (status, result bytes) per frame, input order."""
        q = self.parent.queue
        n = len(frames)
        ids = [uuid.uuid4().bytes for _ in frames]
        offsets = np.zeros(n + 1, np.uint64)
        np.cumsum([len(f) for f in frames], out=offsets[1:])
        blob = np.frombuffer(b"".join(frames), np.uint8) if n else np.zeros(0, np.uint8)
        q.push_batch(np.frombuffer(b"".join(ids), np.uint8).reshape(-1, 16), blob, offsets, flags=np.full(n, TF_PICKLE, np.uint8))
        want = {i: k for k, i in enumerate(ids)}
        out: List[Optional[Tuple[str, Optional[bytes]]]] = [None] * n
        cb = bool(self.parent.callback_url)
        if cb and not self.parent._cb_set:
            q.set_callback_policy(self.parent.signing_key)
            q.set_callback_runners(function=True)
            self.parent._cb_set = True
        self.callbacks = [None] * n
        seen = 0
        while seen < n:
            r = q.drain(self.parent.gpu_handler, full_pickle=self.parent.full_pickle, callbacks=cb)
            if r.n == 0:
                break
            for i in range(r.n):
                k = want.get(r.task_ids[i].tobytes())
                if k is not None:
                    out[k] = (STATUS_NAMES[int(r.status[i])], r.result(i))
                    if cb and int(r.cb_kind[i]) == L.CB_POST:
                        self.callbacks[k] = (r.callback_url(i) or self.parent.callback_url, r.callback_body(i), r.callback_headers(i))
                    seen += 1
        return [o if o is not None else ("ERROR", None) for o in out]

    def _call_remote(self, *args: Any, **kwargs: Any) -> Any:
        status, res = self._run_batch([self._frame(args, kwargs)])[0]
        if status == "UNSUPPORTED":
            self.unsupported.append((args, kwargs))
        if status != "COMPLETE" or not res:                       # function.py:223-231: failed -> None; empty result -> None
            return None
        return cloudpickle.loads(res)

    def map(self, inputs: Sequence[Any]) -> Iterator[Any]:
        """function.py:253-282: one task per input; yields one result per input (None for a failed task). The reference
        yields in completion order (as_completed, :260); here that is the order of the records."""
        if not self.parent.prepare_runtime(func=self.func, stub_type=self.base_stub_type):
            return
        inputs = list(inputs)
        frames = [self._frame(tuple(self._format_args(x)), {}) for x in inputs]
        for x, (status, res) in zip(inputs, self._run_batch(frames)):
            if status == "UNSUPPORTED":
                self.unsupported.append(x)
            yield cloudpickle.loads(res) if status == "COMPLETE" and res else None


def function(*args: Any, **kwargs: Any) -> Function:
    """`@function(...)` spelling of the decorator."""
    return Function(*args, **kwargs)
