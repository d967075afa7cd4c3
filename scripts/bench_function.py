"""GPU: throughput of the function path with B9_DRAIN_PICKLE_FULL (`.map()` fan-out; no target: these are first numbers).

    python scripts/bench_function.py [--calls K] [--warmup W] [--host-sample N]

Workloads: json_sum over 25 k and 100 k pickled configs[4] documents (synth.function_docs_batch), identity over 100 k
pickled synth.values_batch values, crc32 over 1 M pickled zipf strings (synth.crc_batch's strings). Each resident batch is
drained K times with B9_DRAIN_PEEK | B9_DRAIN_PICKLE_FULL (nothing is consumed); the time of a call is the kernel time
b9_stats reports for it (CUDA events around drain3_kernel and the pickle pass), the median of K. In the same run the
reference runner loop (cloudpickle.loads -> handler -> cloudpickle.dumps, oracle/pyoracle/funcloop.py) is timed on one
host core over a sample of each batch; the line states the core count, so a whole-box CPU rate is at most that many times
the per-core one. Prints one JSON line per workload with the card's name and power limit, read in the same run. Writes
nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_wire import card  # noqa: E402


def blobs_of(batch):
    raw = batch.payload.tobytes()
    return [raw[int(batch.offsets[i]):int(batch.offsets[i + 1])] for i in range(batch.n)]


def host_rate(blobs, handler: str, sample: int) -> float:
    from oracle.pyoracle import funcloop
    idx = np.linspace(0, len(blobs) - 1, min(sample, len(blobs))).astype(int)
    t0 = time.perf_counter()
    for i in idx:
        funcloop.run_function_task(blobs[i], handler)
    return len(idx) / (time.perf_counter() - t0)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--host-sample", type=int, default=5000)
    a = ap.parse_args()
    import cloudpickle
    from beta9_b200 import synth
    from beta9_b200.device_queue import DeviceQueue
    info = card()
    crc = synth.crc_batch(1_000_000)
    craw = crc.payload.tobytes()
    crc_blobs = [cloudpickle.dumps({"args": (json.loads(craw[int(crc.offsets[i]):int(crc.offsets[i + 1])])["args"][0],), "kwargs": {}})
                 for i in range(crc.n)]
    vb = synth.values_batch(100_000)
    vraw = vb.payload.tobytes()
    val_blobs = [cloudpickle.dumps({"args": (json.loads(vraw[int(vb.offsets[i]):int(vb.offsets[i + 1])])["args"][0],), "kwargs": {}})
                 for i in range(vb.n)]
    loads = [("json_sum", "function_docs_25k", blobs_of(synth.function_docs_batch(25_000))),
             ("json_sum", "function_docs_100k", blobs_of(synth.function_docs_batch(100_000))),
             ("identity", "function_values_100k", val_blobs),
             ("crc32", "function_zipf_strings_1m", crc_blobs)]
    with DeviceQueue(ring_bytes=1 << 31, ring_tasks=1 << 21, max_drain_tasks=1 << 21, max_result_bytes=1 << 30) as dq:
        for handler, name, blobs in loads:
            b = synth.from_payloads(blobs, name=name)
            dq.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, 0x04, np.uint8))
            ms = []
            for k in range(a.warmup + a.calls):
                dq.drain_launch(handler, peek=True, full_pickle=True)
                if k >= a.warmup:
                    ms.append(float(dq.stats().last_drain_kernel_ms))
            r = dq.fetch()
            assert r.n == b.n
            t = float(np.median(ms)) * 1e-3
            per_core = host_rate(blobs, handler, a.host_sample)
            print(json.dumps({"workload": name, "handler": handler, "tasks": b.n, "calls": a.calls, "kernel_ms_median": 1e3 * t,
                              "kernel_ms_min": min(ms), "tasks_per_sec": b.n / t, "answered": int((r.status != 4).sum()),
                              "unsupported": int((r.status == 4).sum()), "host_loop_tasks_per_sec_per_core": per_core,
                              "host_cores": os.cpu_count(), **info}), flush=True)
            dq.drain(handler, max_tasks=b.n)
            assert dq.depth() == 0


if __name__ == "__main__":
    main()
