"""GPU: cost of the retry policy's re-push (b9_set_retry_policy). Not a BASELINE config; no target.

    python scripts/bench_retry.py [--tasks N] [--reps R]

N (default 1 Mi) json_sum tasks of configs[4]'s shape (4096 distinct synth.json_batch documents of 256 bytes, repeated
under N ids), of which a fraction f in {1 %, 100 %} has no "values" key (KeyError). For each f the same window is
drained R times with the policy
retry_for=[KeyError] (those tasks come back RETRY and are pushed again at the fetch) and R times without one (they come
back ERROR), alternated, on the same ctx:
  - drain_ms: b9_drain of the whole window, host clock around the call, which ends in a stream synchronise: kernel,
    read-back and commit; with the policy the commit includes the re-push (gather, scan, copy, slot words);
  - repush_ns_per_task: (median retry drain - median error drain) / retried tasks.
Between two timed drains the re-pushed tasks are drained away untimed. Prints one JSON line per f with the card's name
and power limit. Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_cancel import card  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tasks", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    from beta9_b200 import synth
    from beta9_b200.device_queue import DeviceQueue
    info = card()
    distinct = synth.json_batch(4096, doc_bytes=256, seed=61).tasks()       # (json_batch builds ~2 k documents/s)
    docs = [distinct[i % len(distinct)] for i in range(a.tasks)]
    with DeviceQueue(ring_bytes=1 << 30, ring_tasks=1 << 21, max_drain_tasks=1 << 21, max_result_bytes=1 << 28) as dq:
        for frac in (0.01, 1.0):
            rng = np.random.default_rng(int(frac * 1000))
            bad = rng.random(len(docs)) < frac
            payloads = [d.replace(b'"values"', b'"valuez"', 1) if bad[i] else d for i, d in enumerate(docs)]
            b = synth.from_payloads(payloads, seed=62)
            n_bad = int(bad.sum())
            times = {"retry": [], "error": []}
            for rep in range(a.reps + 1):                                  # (rep 0 warms both paths up)
                for mode in ("retry", "error"):
                    dq.set_retry_policy([KeyError] if mode == "retry" else [], 255)
                    dq.push_batch(b.task_ids, b.payload, b.offsets)
                    dq.sync()
                    t0 = time.perf_counter()
                    r = dq.drain("json_sum", b.n)
                    dt = time.perf_counter() - t0
                    assert r.n_popped == b.n
                    st = np.bincount(r.status, minlength=6)
                    assert st[2 if mode == "retry" else 1] == n_bad, st
                    assert dq.depth() == (n_bad if mode == "retry" else 0)
                    if rep:
                        times[mode].append(dt)
                    dq.set_retry_policy([], 255)
                    while dq.depth():
                        dq.drain("json_sum", b.n)
            mr, me = statistics.median(times["retry"]), statistics.median(times["error"])
            print(json.dumps({"tasks": b.n, "retried": n_bad, "frac": frac, "reps": a.reps,
                              "drain_retry_ms": 1e3 * mr, "drain_error_ms": 1e3 * me,
                              "drain_retry_ms_min": 1e3 * min(times["retry"]), "drain_error_ms_min": 1e3 * min(times["error"]),
                              "repush_ns_per_task": 1e9 * (mr - me) / max(1, n_bad), **info}), flush=True)


if __name__ == "__main__":
    main()
