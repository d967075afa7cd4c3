"""GPU: cost of b9_cancel (StopTasks by id) over a full ring, and of the drain after it. Not a BASELINE config; no target.

    python scripts/bench_cancel.py [--tasks N] [--reps R] [--steps K] [--warmup W]

N (default 4 Mi) pending configs[1]-shaped tasks (synth.strings_batch(N, 256), 1 % needing escapes). For each request
size n in {1, 1 Ki, 64 Ki, 1 Mi} ids, half of them pending tasks and half unknown, the queue is filled afresh and:
  - drain_clean_ms: K peek drains of the whole window with nothing cancelled, device time as bench.py takes it;
  - sort_ms: b9_cancel of the request on an empty queue: the host sort and de-duplication, which run before the call
    looks at the ring (median of R calls, host clock);
  - cancel_ms: b9_cancel of R different requests of n ids over the full ring, host clock around each call, which ends
    in a stream synchronise: sort + key upload + cancel_kernel + outcome read-back (median of R);
  - drain_after_ms: K peek drains of the same window once R * n / 2 tasks are cancelled: the count pre-pass path.
The kernel reads 16 B of id per slot and 8 B of header per hit: floor_us is those bytes at the data sheet's 3.35 TB/s.
Prints one JSON line per n with the card's name and power limit. Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": out[0].strip(), "power_limit_w": float(out[1])}
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        return {"gpu": None, "power_limit_w": None}


def peek_ms(dq, n: int, steps: int, warmup: int) -> float:
    for _ in range(warmup):
        dq.drain_launch("identity", n, peek=True)
    for _ in range(steps):
        dq.drain_launch("identity", n, peek=True, wait=False)
    dq.sync()
    return float(dq.stats().last_drain_kernel_ms) / steps


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tasks", type=int, default=1 << 22)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    from beta9_b200 import synth
    from beta9_b200.device_queue import DeviceQueue
    info = card()
    q4 = a.tasks // 4                              # (four seeds: one strings_batch of 4 Mi would need 8 GB of draws)
    b = synth.concat([synth.strings_batch(q4 if k < 3 else a.tasks - 3 * q4, 256, seed=synth.SEED + k) for k in range(4)])
    rng = np.random.default_rng(7)
    with DeviceQueue(ring_bytes=1 << 31, ring_tasks=1 << 22, max_drain_tasks=1 << 22, max_result_bytes=1 << 31) as dq, \
            DeviceQueue(ring_bytes=1 << 20, ring_tasks=1 << 10, max_drain_tasks=1 << 10, max_result_bytes=1 << 20) as empty:
        for n in (1, 1 << 10, 1 << 16, 1 << 20):
            present = (n + 1) // 2
            assert present * a.reps <= b.n, "fewer pending tasks than the requests cancel"
            picks = rng.permutation(b.n)[:present * a.reps].reshape(a.reps, present)
            reqs = []
            for k in range(a.reps):
                req = np.concatenate([b.task_ids[picks[k]], synth.task_ids(n - present, seed=1000 + k)])
                reqs.append(np.ascontiguousarray(req[rng.permutation(n)]))
            dq.push_batch(b.task_ids, b.payload, b.offsets)
            clean = peek_ms(dq, b.n, a.steps, a.warmup)
            empty.cancel(reqs[0])
            sort_s, cancel_s, marked = [], [], 0
            for req in reqs:
                t0 = time.perf_counter(); empty.cancel(req); sort_s.append(time.perf_counter() - t0)
            for req in reqs:
                t0 = time.perf_counter(); m, _ = dq.cancel(req); cancel_s.append(time.perf_counter() - t0)
                assert m == present, (m, present)
                marked += m
            after = peek_ms(dq, b.n, a.steps, a.warmup)
            r = dq.drain("identity", b.n)
            assert r.n_popped == b.n and r.n == b.n - marked and dq.depth() == 0
            floor_bytes = 16 * b.n + 8 * present
            print(json.dumps({"ids": n, "present": present, "pending": b.n, "reps": a.reps,
                              "sort_ms": 1e3 * statistics.median(sort_s), "cancel_ms": 1e3 * statistics.median(cancel_s),
                              "cancel_ms_min": 1e3 * min(cancel_s), "floor_us": 1e6 * floor_bytes / HBM_BYTES_PER_S,
                              "drain_clean_ms": clean, "drain_after_ms": after, "cancelled_in_window": marked, **info}), flush=True)


if __name__ == "__main__":
    main()
