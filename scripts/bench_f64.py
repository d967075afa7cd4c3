"""GPU: throughput of the float64 / container legs, which are not BASELINE configs and have no target.

    python scripts/bench_f64.py [--steps K] [--warmup W] [--identity-tasks N] [--json-tasks N]

Times identity over synth.values_batch (SDK payloads of numbers, nested lists and dicts) and json_sum over
synth.json_float_batch (configs[4]'s 1 KB document shape with float64 values), the way bench.py times a drain:
K peek launches enqueued back to back, device time from the CUDA events on the drain stream. Prints one JSON line per
leg, with the card's name and power limit. Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": out[0].strip(), "power_limit_w": float(out[1])}
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        return {"gpu": None, "power_limit_w": None}


def leg(dq, batch, handler: str, steps: int, warmup: int) -> dict:
    n = batch.n
    dq.push_batch(batch.task_ids, batch.payload, batch.offsets)
    for _ in range(warmup):
        dq.drain_launch(handler, n, peek=True)
    for _ in range(steps):
        got = dq.drain_launch(handler, n, peek=True, wait=False)
    dq.sync()
    dev_s = float(dq.stats().last_drain_kernel_ms) * 1e-3
    assert got == n, (got, n)
    dq.drain_launch(handler, n, peek=False)
    res = dq.fetch()
    assert res.n == n and dq.depth() == 0
    unsupported = int((res.status == 4).sum())
    return {"handler": handler, "workload": batch.name, "tasks": n, "steps": steps, "tasks_per_sec": n * steps / dev_s,
            "ms_per_step": 1e3 * dev_s / steps, "unsupported": unsupported, "payload_bytes_per_task": batch.payload.size / n}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--identity-tasks", type=int, default=100_000)
    ap.add_argument("--json-tasks", type=int, default=25_000, help="default: configs[4]'s tasks per GPU")
    a = ap.parse_args()
    from beta9_b200 import synth
    from beta9_b200.device_queue import DeviceQueue
    info = card()
    legs = [(synth.values_batch(a.identity_tasks), "identity"), (synth.json_float_batch(a.json_tasks), "json_sum")]
    with DeviceQueue(ring_bytes=1 << 30, ring_tasks=1 << 21, max_drain_tasks=1 << 21, max_result_bytes=1 << 30) as dq:
        for batch, handler in legs:
            print(json.dumps({**leg(dq, batch, handler, a.steps, a.warmup), **info}), flush=True)


if __name__ == "__main__":
    main()
