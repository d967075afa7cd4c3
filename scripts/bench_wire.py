"""GPU: throughput of the device TaskMessage encoder, b9_wire_encode and b9_wire_encode_full (no BASELINE config, no target).

    python scripts/bench_wire.py [--calls K] [--warmup W]

Workloads: configs[1] (1 M x 256-char strings, 1 % needing escapes), configs[4]'s shape (synth.json_batch, 100 k
{"id", "values", "pad"} documents: keys not in Go's order), synth.json_float_batch (20 k) and synth.values_batch (100 k).
Both entry points run K times over each resident batch (the calls are peeks: nothing is consumed); the time of a call is
the kernel time b9_stats reports for it (CUDA events around the kernel), the median of K. Prints one JSON line per
(workload, entry point) with tasks/s (all tasks of the window, encoded or declined), record GB/s (record bytes written),
the answered and UNSUPPORTED counts and the card's name and power limit, read in the same run. Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": out[0].strip(), "power_limit_w": float(out[1])}
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        return {"gpu": None, "power_limit_w": None}


def leg(dq, batch, full: bool, calls: int, warmup: int) -> dict:
    ms = []
    for k in range(warmup + calls):
        r = dq.wire_encode("ws-b200", "7f1c2d3e-4a5b-4c6d-8e9f-0a1b2c3d4e5f", full=full)
        if k >= warmup:
            ms.append(float(dq.stats().last_drain_kernel_ms))
    assert r.n == batch.n
    t = float(np.median(ms)) * 1e-3
    out_bytes = int(r.lengths.astype(np.int64).sum())
    return {"entry": "b9_wire_encode_full" if full else "b9_wire_encode", "workload": batch.name, "tasks": batch.n, "calls": calls,
            "kernel_ms_median": 1e3 * t, "kernel_ms_min": min(ms), "tasks_per_sec": batch.n / t, "record_gb_per_sec": out_bytes / t / 1e9,
            "answered": int((r.status == 0).sum()), "unsupported": int((r.status == 4).sum()), "record_bytes": out_bytes}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    assert a.calls >= 10
    from beta9_b200 import synth
    from beta9_b200.device_queue import DeviceQueue
    info = card()
    loads = [synth.strings_batch(1_000_000, 256), synth.json_batch(100_000), synth.json_float_batch(20_000), synth.values_batch(100_000)]
    with DeviceQueue(ring_bytes=1 << 31, ring_tasks=1 << 20, max_drain_tasks=1 << 20, max_result_bytes=3 << 30) as dq:
        for batch in loads:
            dq.push_batch(batch.task_ids, batch.payload, batch.offsets)
            for full in (False, True):
                print(json.dumps({**leg(dq, batch, full, a.calls, a.warmup), **info}), flush=True)
            dq.drain("identity", max_tasks=batch.n)
            assert dq.depth() == 0


if __name__ == "__main__":
    main()
