"""Host-side mirror of the reference's Python surface for this path — same names, argument meaning
and error behaviour, with the per-task gRPC round trips replaced by the batch C ABI.

  TaskQueue / _CallableWrapper.put     sdk/src/beta9/abstractions/taskqueue.py:130-158,254-295
  Function-style .map()                sdk/src/beta9/abstractions/function.py:253-282
  TaskQueueWorker.process_tasks        sdk/src/beta9/runner/taskqueue.py:297-404 (pop -> handler -> complete)
  RedisTaskQueue.put admission         pkg/abstractions/taskqueue/taskqueue.go:176-208 (max_pending_tasks)

The user function is kept for `.local()` and for calling the wrapper inside a container, exactly as
in the reference; remote execution runs the stub's GPU kernel handler (`gpu_handler=`). There is no
CPU fallback: tasks the device handler does not implement come back with status "UNSUPPORTED".
"""
from __future__ import annotations

import base64
import hashlib
import hmac
import json
import os
import uuid
from dataclasses import dataclass
from typing import Any, Callable, Dict, Iterator, List, Optional, Sequence, Union

import numpy as np

from . import _lib as L
from .device_queue import DeviceQueue, STATUS_NAMES

TASKQUEUE_STUB_TYPE = "taskqueue"
DEFAULT_MAX_PENDING_TASKS = 100      # sdk/src/beta9/abstractions/taskqueue.py:142
_CANCEL_MAX_IDS = 1 << 20            # most ids one b9_cancel takes


@dataclass
class Task:
    """What `put()` hands back (the reference returns the REST client's Task for `task_id`)."""
    id: str
    status: str = "PENDING"
    result: Any = None
    result_bytes: Optional[bytes] = None
    # with a stub callback_url: what the runner hands requests.post after this task, (url, body bytes, headers); None
    # where it posts nothing (RETRY, a body requests refuses) or where the device did not settle the task (UNSUPPORTED)
    callback: Optional[tuple] = None

    def raw_id(self) -> bytes:
        return uuid.UUID(self.id).bytes


class TaskQueue:
    """Decorator. Resource arguments are accepted and kept for API compatibility; only the ones
    this path reads have an effect (`max_pending_tasks`, `retries`, `retry_for`, `gpu_handler`, `gpu_handler_image`,
    `device`). A task whose
    handler raises a class in `retry_for` (an exact match, as the runner's retry_on_errors) comes back "RETRY" and is
    queued again, up to `retries` times; after that it comes back "RETRY_LIMIT" (the gateway cancels it). With
    `callback_url`, every drained task carries the callback the runner would post (Task.callback), signed with the
    workspace's `signing_key` (None or b"": unsigned, as a gateway without a key); nothing is posted here."""

    def __init__(self, cpu: Union[int, float, str] = 1.0, memory: Union[int, str] = 128, gpu: Any = "", image: Any = None,
                 timeout: int = 3600, retries: int = 3, workers: int = 1, keep_warm_seconds: int = 10,
                 max_pending_tasks: int = DEFAULT_MAX_PENDING_TASKS, name: Optional[str] = None,
                 retry_for: Optional[List[type]] = None, gpu_handler: Optional[str] = None, device: int = 0, queue: Optional[DeviceQueue] = None,
                 gpu_handler_image: Optional[Union[bytes, str]] = None,
                 callback_url: Optional[str] = None, signing_key: Optional[bytes] = None, **kwargs: Any):
        self.cpu = int(float(cpu) * 1000) if not isinstance(cpu, str) else cpu     # base/runner.py parse_cpu: cores -> millicores
        self.memory = memory
        self.gpu = gpu
        self.image = image
        self.timeout = timeout
        self.retries = retries
        self.retry_for = list(retry_for or [])
        self.callback_url = callback_url
        self.signing_key = bytes(signing_key or b"")
        self.workers = workers
        self.keep_warm_seconds = keep_warm_seconds
        self.max_pending_tasks = max_pending_tasks
        self.name = name
        self.gpu_handler = gpu_handler or os.environ.get("B9_GPU_HANDLER", "identity")
        # a user handler (b9gpu_handler.cuh): the sm_90a image (bytes or a path) that holds B9_HANDLER(gpu_handler, ...)
        self.gpu_handler_image = gpu_handler_image or os.environ.get("B9_GPU_HANDLER_IMAGE") or None
        self._handler_loaded = False
        self.device = device
        self.extra = kwargs
        self._queue = queue
        self._policy_set = False
        self.stub_id = str(uuid.uuid4())

    @property
    def queue(self) -> DeviceQueue:
        if self._queue is None:
            self._queue = DeviceQueue(device=self.device)     # raises without a GPU: no CPU path
        if self.gpu_handler_image is not None and not self._handler_loaded:
            self._queue.load_handler(self.gpu_handler_image, self.gpu_handler)
            self._handler_loaded = True
        if not self._policy_set:
            self._queue.set_retry_policy(self.retry_for, self.retries)
            if self.callback_url:
                self._queue.set_callback_policy(self.signing_key)
            self._policy_set = True
        return self._queue

    def prepare_runtime(self, func: Optional[Callable] = None, stub_type: str = TASKQUEUE_STUB_TYPE) -> bool:
        # the reference creates/syncs the stub here (base/runner.py); nothing to upload for a kernel handler
        return True

    def __call__(self, func: Callable) -> "_CallableWrapper":
        return _CallableWrapper(func, self)


class _CallableWrapper:
    def __init__(self, func: Callable, parent: TaskQueue):
        self.func = func
        self.parent = parent
        self._held: List[Task] = []       # drained on behalf of a map(): handed out by the next process_tasks()
        self._cb_override: Dict[str, Any] = {}   # task id -> its "callback_url" kwarg (the device leaves those to the host)

    def __call__(self, *args: Any, **kwargs: Any) -> Any:
        # sdk taskqueue.py:218-224: callable only inside a container
        if os.environ.get("CONTAINER_ID") is not None:
            return self.local(*args, **kwargs)
        raise NotImplementedError("Direct calls to TaskQueues are not supported. Please use the `put` method.")

    def local(self, *args: Any, **kwargs: Any) -> Any:
        return self.func(*args, **kwargs)

    # ---- producer
    @staticmethod
    def _payload(args: Sequence[Any], kwargs: dict) -> bytes:
        return json.dumps({"args": args, "kwargs": kwargs}).encode("utf-8")       # taskqueue.py:284-285

    def put(self, *args: Any, **kwargs: Any) -> Union[bool, Task]:
        """Enqueue one task (a batch of one). Returns a Task, or False when the queue refuses it
        (`Failed to enqueue task`: admission limit or ring full), like the reference."""
        r = self.put_batch([(args, kwargs)])
        return r[0] if r else False

    def put_batch(self, calls: Sequence[Any]) -> List[Task]:
        """Enqueue many tasks with ONE push. `calls` items are (args, kwargs) pairs, or bare args
        tuples / single values (formatted like Function.map's inputs, function.py:246-251)."""
        if not self.parent.prepare_runtime(func=self.func, stub_type=TASKQUEUE_STUB_TYPE):
            return []
        q = self.parent.queue
        norm = [self._normalise(c) for c in calls]
        if not norm:
            return []
        # RedisTaskQueue.put: tasksInFlight >= MaxPendingTasks -> ErrExceededTaskLimit (taskqueue.go:182-189);
        # a batch is admitted only as a whole
        if q.depth() + len(norm) > self.parent.max_pending_tasks:
            return []
        payloads = [self._payload(a, k) for a, k in norm]
        ids = [uuid.uuid4() for _ in norm]
        if self.parent.callback_url:
            self._cb_override.update((str(i), k["callback_url"]) for i, (_, k) in zip(ids, norm) if "callback_url" in k)
        offsets = np.zeros(len(norm) + 1, np.uint64)
        np.cumsum([len(p) for p in payloads], out=offsets[1:])
        blob = np.frombuffer(b"".join(payloads), np.uint8)
        id_arr = np.frombuffer(b"".join(i.bytes for i in ids), np.uint8).reshape(-1, 16)
        try:
            q.push_batch(id_arr, blob, offsets)
        except Exception as e:                                # ring full etc. -> ok=false
            if getattr(e, "code", None) in (-28, -7):
                return []
            raise
        return [Task(id=str(i)) for i in ids]

    @staticmethod
    def _format_args(args: Any) -> List[Any]:
        """sdk/src/beta9/abstractions/function.py:246-251."""
        if isinstance(args, tuple):
            return list(args)
        if not isinstance(args, list):
            return [args]
        return args

    @staticmethod
    def _normalise(c: Any):
        if isinstance(c, tuple) and len(c) == 2 and isinstance(c[0], (tuple, list)) and isinstance(c[1], dict):
            return tuple(c[0]), c[1]
        if isinstance(c, tuple):
            return c, {}
        if isinstance(c, list):
            return tuple(c), {}
        return (c,), {}

    def stop_tasks(self, task_ids: Sequence[str]) -> Dict[str, str]:
        """The gateway's StopTasks (pkg/api/v1/task.go:333-398) for this queue: every pending task with one of these ids is
        cancelled and produces no record. Per id: "CANCELLED", "ALREADY_CANCELLED", "RUNNING" (claimed by a drain in flight:
        left alone) or "NOT_FOUND"; ids that are unknown or not UUIDs are ignored, as the reference ignores them."""
        names = {str(t): "NOT_FOUND" for t in task_ids}
        raw = []
        for t in names:
            try:
                raw.append((t, uuid.UUID(t).bytes))
            except ValueError:
                continue
        q = self.parent.queue
        for lo in range(0, len(raw), _CANCEL_MAX_IDS):
            part = raw[lo:lo + _CANCEL_MAX_IDS]
            ids = np.frombuffer(b"".join(b for _, b in part), np.uint8).reshape(-1, 16)
            _, outcome = q.cancel(ids)
            for (t, _), o in zip(part, outcome):
                names[t] = ("CANCELLED" if o & L.CANCEL_MARKED else "ALREADY_CANCELLED" if o & L.CANCEL_ALREADY
                            else "RUNNING" if o & L.CANCEL_CLAIMED else "NOT_FOUND")
        return names

    # ---- consumer (what the runner loop + TaskQueueComplete hand back)
    def process_tasks(self, max_tasks: int = 1 << 22) -> List[Task]:
        """Drain up to max_tasks pending tasks through the kernel handler; FIFO order. Tasks that a `map()` had to drain
        on the way to its own (they were queued before it) are handed out first: nothing is dropped."""
        out, self._held = self._held[:max_tasks], self._held[max_tasks:]
        if len(out) < max_tasks:
            out += self._drain(max_tasks - len(out))
        return out

    def _drain(self, max_tasks: int) -> List[Task]:
        cb = bool(self.parent.callback_url)
        q = self.parent.queue
        res = q.drain(self.parent.gpu_handler, max_tasks=max_tasks, callbacks=True) if cb else q.drain(self.parent.gpu_handler, max_tasks=max_tasks)
        out = []
        for i in range(res.n):
            rb = res.result(i)
            t = Task(id=str(uuid.UUID(bytes=res.task_ids[i].tobytes())), status=STATUS_NAMES[int(res.status[i])],
                     result=json.loads(rb) if rb is not None else None, result_bytes=rb)
            if cb:
                t.callback = self._callback(res, i, t)
            out.append(t)
        return out

    def _callback(self, res, i: int, t: Task) -> Optional[tuple]:
        """send_callback's request for record i (runner/common.py:430-481): the device's signature for B9_CB_POST; the one
        kind the host settles here is an ERROR whose kwargs carried "callback_url" (the runner's override), signed on the
        CPU as SignPayload does (pkg/auth/sign.go:17-35)."""
        kind = int(res.cb_kind[i])
        override = self._cb_override.pop(t.id, None)
        if kind == L.CB_POST:
            return self.parent.callback_url, res.callback_body(i), res.callback_headers(i)
        if kind == L.CB_HOST and t.status == "ERROR":
            url = override or self.parent.callback_url
            body = res.callback_body(i)
            key, ts = self.parent.signing_key, res.cb_timestamp
            sig = hmac.new(key, base64.b64encode(body) + b":%d" % ts, hashlib.sha256).hexdigest() if key else ""
            headers = res.callback_headers(i)
            headers["X-Task-Signature"] = sig
            return url, body, headers
        return None

    def map(self, inputs: Sequence[Any]) -> Iterator[Any]:
        """Fan out: one task per input, one push, then drains until every one of ITS tasks has come back; yields each
        task's result (None for a task that failed or produced no result, as function.py:266-268 does). The queue is
        FIFO: tasks that earlier `put()`s left pending are drained on the way and kept for the next `process_tasks()`."""
        # Function.map spreads each input as positional arguments after `_format_args` (function.py:246-251):
        # a tuple or list IS the argument list, anything else is the single argument; never keyword arguments
        tasks = self.put_batch([(tuple(self._format_args(x)), {}) for x in inputs])
        if len(tasks) != len(inputs):
            raise RuntimeError("Failed to enqueue tasks")
        want = {t.id for t in tasks}
        done = {}
        while len(done) < len(want):
            got = self._drain(1 << 22)
            if not got:
                break                                         # cancelled / expired tasks produce no record: their result is None
            for t in got:
                if t.id in want:
                    if t.status != "RETRY":                   # a retried task is queued again: its answer comes later
                        done[t.id] = t
                else:
                    self._held.append(t)
        for t in tasks:
            yield done[t.id].result if t.id in done else None


def task_queue(*args: Any, **kwargs: Any) -> TaskQueue:
    """`@task_queue(...)` spelling of the decorator (sdk/src/beta9/__init__.py exports both)."""
    return TaskQueue(*args, **kwargs)
