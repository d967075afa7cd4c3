"""The task loop with a stub's `retry_for` / `retries` (TaskPolicy.MaxRetries): oracle.pyoracle.loop.run_task_loop's
push and runner halves, plus what happens when the handler raises a class the stub retries on.

  runner   sdk/src/beta9/runner/taskqueue.py:352-393,407-408  TaskStatus.Retry when retry_on_errors(retry_for, e):
                                                              `type(e) is err`, an exact class match; result None
  gateway  pkg/abstractions/taskqueue/taskqueue.go:360-363,680-710, pkg/task/dispatch.go:232-285
                                                              RetryTask: Retries < MaxRetries -> Retries += 1,
                                                              Timestamp = now, re-encode, RPUSH at the tail; otherwise
                                                              the task is cancelled (TaskExceededRetryLimit): RETRY_LIMIT

The runner half calls the same functions in the same order as the reference and is pinned against the reference's own
TaskQueueWorker.process_tasks by tests/golden/make_ref_retry_golden.py (tests/test_retry_on_host.py). The gateway half is
a restatement of Go code (PARITY UNPINNED: there is no Go toolchain here), like the Go halves in oracle/pyoracle.
Shared by the CPU and GPU tests of the retry policy."""
from __future__ import annotations

import json
from collections import deque
from dataclasses import dataclass
from typing import Any, Callable, List, Optional, Sequence

from oracle.pyoracle.gojson import GoJSONError, go_unmarshal_task_payload
from oracle.pyoracle.handlers import HANDLERS
from oracle.pyoracle.httpserialize import InvalidRequestPayload, serialize_http_payload
from oracle.pyoracle.loop import COMPLETE, ERROR, REJECTED, RETRY, serialize_result
from oracle.pyoracle.wire import QueueEnv, build_task_message, format_uuid

# Not a runner status: the runner reported Retry, but the task had used up Policy.MaxRetries, so RetryTask cancels it
# with TaskExceededRetryLimit instead of re-queueing it (B9_ST_RETRY_LIMIT).
RETRY_LIMIT = "RETRY_LIMIT"


@dataclass
class Answer:
    task_id: bytes              # raw 16-byte uuid
    status: str
    result: Optional[bytes]     # TaskQueueCompleteRequest.result; None = unset
    exc: Optional[type] = None  # ERROR / RETRY / RETRY_LIMIT: type(e) of what the handler raised


def retry_on_errors(retry_for: Sequence[type], e: BaseException) -> bool:
    """sdk/src/beta9/runner/taskqueue.py:407-408."""
    return any([err for err in retry_for if type(e) is err])


def call_handler(fn: Callable[..., Any], args, kwargs, retry_for: Sequence[type]):
    """runner/taskqueue.py:349-378: (status, result bytes or None, type(e) or None)."""
    status, result, exc = COMPLETE, None, None
    try:
        result = fn(*(args or []), **(kwargs or {}))
    except BaseException as e:
        exc = type(e)
        status = RETRY if retry_on_errors(retry_for, e) else ERROR
    return status, (serialize_result(result) if result else None), exc


def run_retry_loop(payloads: Sequence[bytes], task_ids: Sequence[bytes], handler: "str | Callable[..., Any]",
                   retry_for: Sequence[type] = (), max_retries: int = 3, retries: Optional[Sequence[int]] = None,
                   http_body: Sequence[bool] = (), task_msg: Sequence[bool] = (), env: Optional[QueueEnv] = None,
                   now_unix_ns: int = 1_789_970_992_573_161_412) -> List[Answer]:
    """Push every payload in order, then drain the queue FIFO through one runner until it is empty. Returns every answer
    in the order the runner gave them (a retried task answers once per attempt). A payload the gateway refuses is
    REJECTED at its place in the FIFO order, where the device's drain reports it. http_body[i] / task_msg[i]: payload i is an HTTP body (SerializeHttpPayload) / a TaskMessage record already
    (the runner json.loads it as it is). `retries[i]`: task i's Retries at the push (0 by default)."""
    env = env or QueueEnv()
    fn = HANDLERS[handler] if isinstance(handler, str) else handler
    out: List[Answer] = []
    queue: deque = deque()
    for i, (p, tid) in enumerate(zip(payloads, task_ids)):
        p = bytes(p)
        r0 = int(retries[i]) if retries is not None else 0
        if i < len(task_msg) and task_msg[i]:
            queue.append((i, p, r0))
            continue
        try:
            if i < len(http_body) and http_body[i]:
                args, kwargs = serialize_http_payload(p)
            else:
                args, kwargs = go_unmarshal_task_payload(p)
        except (GoJSONError, InvalidRequestPayload):
            queue.append((i, None, r0))
            continue
        queue.append((i, build_task_message(env, format_uuid(tid), args, kwargs, now_unix_ns, retries=r0).encode(), r0))
    while queue:
        i, wire, r = queue.popleft()                                    # LPOP
        if wire is None:
            out.append(Answer(bytes(task_ids[i]), REJECTED, None))
            continue
        task = json.loads(wire)                                         # runner/taskqueue.py:196
        assert task["task_id"] == format_uuid(task_ids[i])
        status, res, exc = call_handler(fn, task["args"], task["kwargs"], retry_for)
        if status == RETRY:
            if r < max_retries:                                         # RetryTask: Retries += 1, RPUSH (the record's bytes
                queue.append((i, wire, r + 1))                          # are re-encoded; the runner reads only id / args / kwargs)
            else:
                status = RETRY_LIMIT
        out.append(Answer(bytes(task_ids[i]), status, res, exc))
    return out
