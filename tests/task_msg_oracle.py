"""The runner's half of the task loop over given TaskMessage records: what TaskQueuePop hands the runner as `task_msg`
(pkg/abstractions/taskqueue/taskqueue.go:238-309) and what the runner does with it -- json.loads, then
handler(*(args or []), **(kwargs or {})), then serialize_result (sdk/src/beta9/runner/taskqueue.py:196-201,349-378).
It is the consumer half of oracle.pyoracle.loop.run_task_loop, with the same stdlib calls in the same order, over
bytes the caller gives. Shared by the CPU and GPU tests of B9_TF_TASK_MSG."""
from __future__ import annotations

import json
from typing import Any, Callable, List, Sequence

from oracle.pyoracle.handlers import HANDLERS
from oracle.pyoracle.loop import COMPLETE, ERROR, TaskResult, serialize_result
from oracle.pyoracle.wire import format_uuid

# Not a reference status: the runner does not get as far as calling the handler on this record (json.loads raises,
# a key is missing, `*args` / `**kwargs` of the wrong type, or a task_id that is not the slot's). The device has to
# report B9_ST_UNSUPPORTED for every such record.
NOT_RUN = "NOT_RUN"


def run_records(records: Sequence[bytes], task_ids: Sequence[bytes],
                handler: "str | Callable[..., Any]") -> List[TaskResult]:
    """task_ids[i] is the raw 16-byte id record i was pushed under."""
    fn = HANDLERS[handler] if isinstance(handler, str) else handler
    results: List[TaskResult] = []
    for wire, tid in zip(records, task_ids):
        wire = bytes(wire)
        try:
            task = json.loads(wire)                     # runner/taskqueue.py:196
            args = task["args"] or []                   # :349-350
            kwargs = task["kwargs"] or {}
            run = task["task_id"] == format_uuid(tid) and isinstance(args, list) and isinstance(kwargs, dict)
        except (ValueError, TypeError, KeyError, RecursionError):
            run = False
        if not run:
            results.append(TaskResult(bytes(tid), NOT_RUN, None, wire))
            continue
        status = COMPLETE
        result = None
        try:
            result = fn(*args, **kwargs)                # :353
        except BaseException:
            status = ERROR                              # :356
        out = serialize_result(result) if result else None   # :378
        results.append(TaskResult(bytes(tid), status, out, wire))
    return results
