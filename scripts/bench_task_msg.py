"""GPU: throughput of draining TaskMessage records (B9_TF_TASK_MSG), which is not a BASELINE config and has no target.

    python scripts/bench_task_msg.py [--steps K] [--warmup W] [--tasks N]

Times identity over N configs[1]-shaped records (the C oracle's TaskMessage.Encode of synth.strings_batch(N, 256):
1 % of the strings need escapes), then the configs[2]-[4] shapes as records: crc32 over 1 M zipf strings, vadd_f32 over
1.25 M vector pairs, json_sum over 25 k documents. Each leg also times the same tasks as SDK payloads. Timing is
bench.py's: K peek launches enqueued back to back, device time from the CUDA events on the drain stream. Prints one
JSON line per leg with tasks/s, ms per step, record bytes per task, the UNSUPPORTED count and the card's name and power
limit. Writes nothing.
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

TF_TASK_MSG = 0x08


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": out[0].strip(), "power_limit_w": float(out[1])}
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        return {"gpu": None, "power_limit_w": None}


def records_of(batch, handler: str):
    """the TaskMessage records the reference would RPUSH for the batch's payloads (C oracle), as a batch"""
    from beta9_b200 import synth
    from oracle import coracle
    o = coracle.run_batch(batch.task_ids, batch.payload, batch.offsets, handler, nthreads=os.cpu_count() or 1, keep_wire=True)
    return synth.Batch(batch.task_ids, np.ascontiguousarray(o.wire, np.uint8)[:int(o.wire_offsets[-1])],
                       np.ascontiguousarray(o.wire_offsets, np.uint64), batch.name + "_records")


def leg(dq, batch, handler: str, steps: int, warmup: int, flags) -> dict:
    n = batch.n
    dq.push_batch(batch.task_ids, batch.payload, batch.offsets, flags=flags)
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
    return {"handler": handler, "workload": batch.name, "records": flags is not None, "tasks": n, "steps": steps,
            "tasks_per_sec": n * steps / dev_s, "ms_per_step": 1e3 * dev_s / steps, "unsupported": int((res.status == 4).sum()),
            "input_bytes_per_task": batch.payload.size / n}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--tasks", type=int, default=1_000_000, help="configs[1]'s tasks per GPU")
    a = ap.parse_args()
    from beta9_b200 import synth
    from beta9_b200.device_queue import DeviceQueue
    info = card()
    legs = [(synth.strings_batch(a.tasks, 256), "identity"), (synth.crc_batch(1_000_000), "crc32"),
            (synth.vadd_batch(1_250_000), "vadd_f32"), (synth.json_batch(25_000), "json_sum")]
    with DeviceQueue(ring_bytes=1 << 32, ring_tasks=1 << 21, max_drain_tasks=1 << 21, max_result_bytes=1 << 30) as dq:
        for batch, handler in legs:
            recs = records_of(batch, handler)
            for b, flags in ((batch, None), (recs, np.full(recs.n, TF_TASK_MSG, np.uint8))):
                print(json.dumps({**leg(dq, b, handler, a.steps, a.warmup, flags), **info}), flush=True)


if __name__ == "__main__":
    main()
