"""GPU: cost of binding a call to a declared signature (B9H_SIGNATURE, examples/handlers greet) on 1 Mi tasks of
256-character strings.

    python scripts/bench_user_signature.py [--reps R]

Three resident windows, each in a context of its own and drained with B9_DRAIN_PEEK:
  - configs[1]'s SDK payloads {"args": [s], "kwargs": {}}: greet called positionally, and echo_str (one Arg, no
    signature), both on this one window;
  - {"args": [], "kwargs": {"name": s, "punct": "?"}}: greet called by keyword;
  - the HTTP body {"name": s}: greet in the endpoint rendering (the body's keys are the kwargs).
The four launches are alternated, R times each after one warm-up of all four. Each figure is the median CUDA-event span
around the launch's kernel (b9_stats.last_drain_kernel_ms). Prints one JSON line per launch kind, with the card's name
and power limit read in the same run. Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_cancel import card  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--tasks", type=int, default=1 << 20)
    a = ap.parse_args()
    assert a.reps >= 7
    from beta9_b200 import _lib as L
    from beta9_b200 import build as B
    from beta9_b200 import synth
    from beta9_b200.device_queue import DeviceQueue
    info = card()
    strs = synth.strings_batch(a.tasks, 256)
    texts = [json.loads(strs.payload[int(strs.offsets[i]):int(strs.offsets[i + 1])].tobytes())["args"][0] for i in range(a.tasks)]
    pos = strs                                                        # {"args": [s], "kwargs": {}}
    kw = synth.from_payloads([json.dumps({"args": [], "kwargs": {"name": t, "punct": "?"}}).encode() for t in texts])
    body = synth.from_payloads([json.dumps({"name": t}).encode() for t in texts])
    windows = ((pos, 0), (kw, 0), (body, L.TF_HTTP_BODY))
    launches = (("greet, positional", 0, "greet", False), ("echo_str, positional", 0, "echo_str", False),
                ("greet, by keyword", 1, "greet", False), ('greet, endpoint body {"name": s}', 2, "greet", True))
    qs = []
    try:
        for b, flags in windows:
            q = DeviceQueue(ring_bytes=1 << 30, ring_tasks=a.tasks, max_drain_tasks=a.tasks, max_result_bytes=1 << 30)
            qs.append(q)
            for h in ("greet", "echo_str"):
                q.load_handler(B.EXAMPLE_CUBIN, h)
            q.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, flags, np.uint8))
            q.sync()
        span = [[] for _ in launches]
        complete = [0] * len(launches)
        for rep in range(a.reps + 1):                                      # (rep 0 warms all four up)
            for k, (label, w, handler, endpoint) in enumerate(launches):
                qs[w].drain_launch(handler, a.tasks, peek=True, endpoint=endpoint)
                if rep:
                    span[k].append(float(qs[w].stats().last_drain_kernel_ms))
                else:
                    complete[k] = int(np.count_nonzero(qs[w].fetch().status == 0))
        for k, (label, w, handler, endpoint) in enumerate(launches):
            line = {"launch": label, "handler": handler, "rendering": "endpoint" if endpoint else "task_queue", "tasks": a.tasks,
                    "complete": complete[k], "reps": a.reps, "kernel_ms": statistics.median(span[k]),
                    "kernel_ms_range": [min(span[k]), max(span[k])]}
            line.update(info)
            print(json.dumps(line), flush=True)
    finally:
        for q in qs:
            q.close()


if __name__ == "__main__":
    main()
