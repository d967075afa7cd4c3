"""GPU: cost of the callback pass (b9_set_callback_policy) on configs[1..4] at their BASELINE size per GPU.

    python scripts/bench_callback.py [--reps R] [--configs 1,2,3,4]

Per workload (the bench.py payloads: configs[1] 1 Mi x 256-char identity strings, configs[2] 1 Mi zipf crc32 strings,
configs[3] 1.25 M vadd_f32 vectors (10 M over 8 GPUs), configs[4] 25 k json_sum documents (100 k over 4 GPUs)), one
resident window drained with B9_DRAIN_PEEK, R times with the policy (a 32-byte key) and R times without, alternated on
the same ctx:
  - drain_ms_plain / drain_ms_signed: the median CUDA-event span around the launch's kernels (b9_stats.last_drain_kernel_ms);
  - sign_kernel_ms: callback_sign_kernel's own time, from torch.profiler's CUDA activity over R signed launches (median);
  - compressions: SHA-256 compressions of the drain, from the record lengths (per record with result bytes R:
    ceil((12 + 4 ceil((len R + 1) / 3) + 1 + digits(ts) + 9) / 64) inner blocks + 1 outer; {"data": {}} is signed once on
    the host), and compressions_per_s = compressions / sign_kernel_ms;
  - added_d2h_bytes: 33 per record (kind + raw digest);
  - cpu_hmac_per_s_one_core: a labelled CPU figure, one core's Python base64 + hmac loop over the same bodies;
  - configs[1] only: e2e_tasks_per_s_signed / _plain, push + drain + fetch of the whole window, host clock, median of R.
Prints one JSON line per workload with the card's name and power limit read in the same run. Writes nothing.
"""
from __future__ import annotations

import argparse
import base64
import hashlib
import hmac
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_cancel import card  # noqa: E402

KEY = b"k" * 32


def workload(cfg: int):
    from beta9_b200 import synth
    if cfg == 1:
        return "identity", synth.strings_batch(1 << 20, 256)
    if cfg == 2:
        return "crc32", synth.crc_batch(1 << 20)
    if cfg == 3:
        return "vadd_f32", synth.vadd_batch(1_250_000)
    return "json_sum", synth.json_batch(25_000)


def compressions(res, ts: int) -> int:
    ln = res.lengths[(res.cb_kind == 1) & (res.has_result == 1)].astype(np.int64)
    q = (ln + 1 + 2) // 3
    inner = (12 + 4 * q + 1 + len(str(ts)) + 9 + 63) // 64
    return int(np.sum(inner + 1))


def sign_kernel_ms(dq, handler: str, n: int, reps: int) -> float:
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            dq.drain_launch(handler, n, peek=True)
        dq.sync()
    times = [e.device_time / 1e3 if hasattr(e, "device_time") else e.cuda_time / 1e3
             for e in prof.events() if "callback_sign_kernel" in e.name]
    del torch
    return statistics.median(times) if times else float("nan")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--configs", default="1,2,3,4")
    a = ap.parse_args()
    from beta9_b200.device_queue import DeviceQueue
    info = card()
    for cfg in [int(x) for x in a.configs.split(",")]:
        handler, b = workload(cfg)
        with DeviceQueue(ring_bytes=1 << 31, ring_tasks=1 << 21, max_drain_tasks=1 << 21, max_result_bytes=1 << 31) as dq:
            dq.push_batch(b.task_ids, b.payload, b.offsets)
            dq.sync()
            span = {"plain": [], "signed": []}
            for rep in range(a.reps + 1):                                  # (rep 0 warms both up)
                for mode in ("plain", "signed"):
                    dq.set_callback_policy(KEY if mode == "signed" else None)
                    dq.drain_launch(handler, b.n, peek=True)
                    if rep:
                        span[mode].append(float(dq.stats().last_drain_kernel_ms))
            dq.set_callback_policy(KEY)
            dq.drain_launch(handler, b.n, peek=True)
            res = dq.fetch(cap_tasks=b.n, callbacks=True)
            comp = compressions(res, res.cb_timestamp)
            k_ms = sign_kernel_ms(dq, handler, b.n, a.reps)
            # one core of the host signing the same bodies with Python's hmac (a sample of up to 100 k)
            sel = np.flatnonzero(res.cb_kind == 1)[:100_000]
            bodies = [res.callback_body(int(i)) for i in sel]
            t0 = time.perf_counter()
            for body in bodies:
                hmac.digest(KEY, base64.b64encode(body) + b":%d" % res.cb_timestamp, hashlib.sha256)
            cpu_rate = len(bodies) / (time.perf_counter() - t0)
            line = {"config": cfg, "handler": handler, "tasks": b.n, "reps": a.reps,
                    "drain_ms_plain": statistics.median(span["plain"]), "drain_ms_signed": statistics.median(span["signed"]),
                    "sign_kernel_ms": k_ms, "compressions": comp, "compressions_per_s": comp / (k_ms * 1e-3) if k_ms == k_ms else None,
                    "kinds": np.bincount(res.cb_kind, minlength=4).tolist(), "added_d2h_bytes": 33 * res.n,
                    "cpu_hmac_per_s_one_core": cpu_rate, "cpu_note": "host CPU, one core, Python base64 + hmac.digest"}
            if cfg == 1:
                e2e = {"plain": [], "signed": []}
                for rep in range(a.reps + 1):
                    for mode in ("plain", "signed"):
                        dq.set_callback_policy(KEY if mode == "signed" else None)
                        while dq.depth():
                            dq.drain(handler, b.n)
                        t0 = time.perf_counter()
                        dq.push_batch(b.task_ids, b.payload, b.offsets)
                        r = dq.drain(handler, b.n, callbacks=mode == "signed")
                        dt = time.perf_counter() - t0
                        assert r.n == b.n
                        if rep:
                            e2e[mode].append(b.n / dt)
                line["e2e_tasks_per_s_plain"] = statistics.median(e2e["plain"])
                line["e2e_tasks_per_s_signed"] = statistics.median(e2e["signed"])
            line.update(info)
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
