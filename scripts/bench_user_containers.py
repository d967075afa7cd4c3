"""GPU: cost of returning lists and dicts from a user handler (the sinks' container calls, examples/handlers tokens and
describe) on configs[1]'s window, 1 Mi SDK payloads {"args": [s], "kwargs": {}} of 256-character strings.

    python scripts/bench_user_containers.py [--reps R] [--parent-image CUBIN]

One resident window for the task-queue rendering and one of the same strings as HTTP bodies for the endpoint rendering,
each in a context of its own and drained with B9_DRAIN_PEEK. echo_str (a string result), tokens (s.split(), a list of
strings) and describe ({"type": "str", "value": s}, a dict with value()) run in both renderings. With --parent-image (an
example image built from an earlier header), its echo_str runs too, beside this build's, so that the string path of
both builds is timed in one run. All launches are alternated, R times each after one warm-up of all. Each figure is the
median CUDA-event span around the launch's kernel (b9_stats.last_drain_kernel_ms). Prints one JSON line per launch
kind, with the card's name and power limit read in the same run. Writes nothing.
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
    ap.add_argument("--parent-image", default=None)
    a = ap.parse_args()
    assert a.reps >= 7
    from beta9_b200 import _lib as L
    from beta9_b200 import build as B
    from beta9_b200 import synth
    from beta9_b200.device_queue import DeviceQueue
    info = card()
    strs = synth.strings_batch(a.tasks, 256)
    texts = [json.loads(strs.payload[int(strs.offsets[i]):int(strs.offsets[i + 1])].tobytes())["args"][0] for i in range(a.tasks)]
    body = synth.from_payloads([json.dumps({"args": [t]}).encode() for t in texts])
    windows = ((strs, 0, False), (body, L.TF_HTTP_BODY, True))
    handlers = ["echo_str", "tokens", "describe"]
    qs, launches = [], []
    try:
        for w, (b, flags, endpoint) in enumerate(windows):
            q = DeviceQueue(ring_bytes=1 << 30, ring_tasks=a.tasks, max_drain_tasks=a.tasks, max_result_bytes=3 << 29)
            qs.append(q)
            ids = {}
            if a.parent_image:
                ids["echo_str (parent build)"] = q.load_handler(a.parent_image, "echo_str")
            for h in handlers:
                ids[h] = q.load_handler(B.EXAMPLE_CUBIN, h)
            q.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, flags, np.uint8))
            q.sync()
            launches += [(label, w, hid, endpoint) for label, hid in ids.items()]
        span = [[] for _ in launches]
        complete = [0] * len(launches)
        for rep in range(a.reps + 1):                                      # (rep 0 warms every launch up)
            for k, (label, w, hid, endpoint) in enumerate(launches):
                qs[w].drain_launch(hid, a.tasks, peek=True, endpoint=endpoint)
                if rep:
                    span[k].append(float(qs[w].stats().last_drain_kernel_ms))
                else:
                    complete[k] = int(np.count_nonzero(qs[w].fetch().status == 0))
        for k, (label, w, hid, endpoint) in enumerate(launches):
            line = {"launch": label, "rendering": "endpoint" if endpoint else "task_queue", "tasks": a.tasks,
                    "complete": complete[k], "reps": a.reps, "kernel_ms": statistics.median(span[k]),
                    "kernel_ms_range": [min(span[k]), max(span[k])]}
            line.update(info)
            print(json.dumps(line), flush=True)
    finally:
        for q in qs:
            q.close()


if __name__ == "__main__":
    main()
