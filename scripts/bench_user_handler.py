"""GPU: cost of a user handler (b9_handler_load, examples/handlers) against the built-in handler it reproduces, at
BASELINE size per GPU.

    python scripts/bench_user_handler.py [--reps R]

Two pairs, each on one resident window drained with B9_DRAIN_PEEK, the user handler's launch and the built-in's alternated
on the same ctx, R times each (after one warm-up of both):
  - crc32_str against crc32 over configs[2]'s 1 Mi zipf strings (32..4096 characters);
  - echo_str against identity over configs[1]'s 1 Mi 256-character strings;
both as task-queue drains (SDK payloads, b9_drain_launch) and as endpoint drains (the same strings as HTTP bodies,
b9_endpoint_drain_launch). Each figure is the median CUDA-event span around the launch's kernel
(b9_stats.last_drain_kernel_ms). Prints one JSON line per pair and rendering, with the card's name and power limit read
in the same run. Writes nothing.
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
    a = ap.parse_args()
    assert a.reps >= 7
    from beta9_b200 import _lib as L
    from beta9_b200 import build as B
    from beta9_b200 import synth
    from beta9_b200.device_queue import DeviceQueue
    info = card()
    pairs = (("configs[2]", synth.crc_batch(1 << 20), "crc32_str", "crc32"),
             ("configs[1]", synth.strings_batch(1 << 20, 256), "echo_str", "identity"))
    with DeviceQueue(ring_bytes=1 << 32, ring_tasks=1 << 21, max_drain_tasks=1 << 21, max_result_bytes=1 << 32) as dq:
        for name in ("crc32_str", "echo_str"):
            dq.load_handler(B.EXAMPLE_CUBIN, name)
        for cfg, b, mine, builtin in pairs:
            for endpoint in (False, True):
                dq.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, L.TF_HTTP_BODY if endpoint else 0, np.uint8))
                dq.sync()
                span = {mine: [], builtin: []}
                for rep in range(a.reps + 1):                              # (rep 0 warms both up)
                    for h in (mine, builtin):
                        dq.drain_launch(h, b.n, peek=True, endpoint=endpoint)
                        if rep:
                            span[h].append(float(dq.stats().last_drain_kernel_ms))
                line = {"config": cfg, "tasks": b.n, "rendering": "endpoint" if endpoint else "task_queue", "reps": a.reps,
                        "user_handler": mine, "user_ms": statistics.median(span[mine]), "user_ms_range": [min(span[mine]), max(span[mine])],
                        "builtin_handler": builtin, "builtin_ms": statistics.median(span[builtin]),
                        "builtin_ms_range": [min(span[builtin]), max(span[builtin])]}
                line["ratio"] = line["user_ms"] / line["builtin_ms"]
                line.update(info)
                print(json.dumps(line), flush=True)
                dq.drain(builtin, b.n, endpoint=endpoint)                # empty the ring for the next window
                assert dq.depth() == 0


if __name__ == "__main__":
    main()
