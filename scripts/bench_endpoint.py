"""GPU: throughput of the endpoint drain (b9_endpoint_drain_launch; no target: these are first numbers).

    python scripts/bench_endpoint.py [--calls K] [--warmup W]

Workloads, every task an HTTP request body (B9_TF_HTTP_BODY): identity over 1 M configs[1] bodies (synth.strings_batch,
256 characters, 1 % with escapes and non-ASCII), crc32 over 1 M zipf strings (synth.crc_batch), json_sum over 100 k
configs[4] documents (synth.json_batch). Each resident batch is drained K times with B9_DRAIN_PEEK by the endpoint drain
and, alternating with it on the same ctx, by the task-queue drain (b9_drain_launch) of the same bodies; the time of a
call is the kernel time b9_stats reports for it (CUDA events around the launch's kernels), the median of K after W
warm-up calls. Prints one JSON line per workload and drain with the card's name and power limit, read in the same run.
Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_wire import card  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    from beta9_b200 import synth
    from beta9_b200.device_queue import DeviceQueue
    info = card()
    loads = [("identity", "configs1_bodies_1m", synth.strings_batch(1_000_000, 256, adversarial_frac=0.01)),
             ("crc32", "zipf_string_bodies_1m", synth.crc_batch(1_000_000)),
             ("json_sum", "configs4_bodies_100k", synth.json_batch(100_000))]
    with DeviceQueue(ring_bytes=1 << 31, ring_tasks=1 << 21, max_drain_tasks=1 << 21, max_result_bytes=1 << 30) as dq:
        for handler, name, b in loads:
            dq.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, 0x02, np.uint8))
            ms = {True: [], False: []}
            for k in range(a.warmup + a.calls):
                for endpoint in (True, False):
                    dq.drain_launch(handler, b.n, peek=True, endpoint=endpoint)
                    if k >= a.warmup:
                        ms[endpoint].append(float(dq.stats().last_drain_kernel_ms))
            for endpoint in (True, False):
                dq.drain_launch(handler, b.n, peek=True, endpoint=endpoint)
                r = dq.fetch()
                assert r.n == b.n
                t = float(np.median(ms[endpoint])) * 1e-3
                print(json.dumps({"workload": name, "handler": handler, "drain": "endpoint" if endpoint else "task_queue",
                                  "tasks": b.n, "calls": a.calls, "kernel_ms_median": 1e3 * t, "kernel_ms_min": min(ms[endpoint]),
                                  "tasks_per_sec": b.n / t, "complete": int((r.status == 0).sum()),
                                  "unsupported": int((r.status == 4).sum()), "out_bytes": int(dq.stats().last_drain_out_bytes),
                                  **info}), flush=True)
            dq.drain(handler, max_tasks=b.n, endpoint=True)
            assert dq.depth() == 0


if __name__ == "__main__":
    main()
