"""GPU: cost of the runners' callback passes (b9_set_callback_runners) at BASELINE size per GPU.

    python scripts/bench_callback_runners.py --runner function|endpoint [--reps R]

function: configs[4]'s 25 k json_sum documents pickled as `.map()` sends them, drained with B9_DRAIN_PICKLE_FULL; endpoint:
configs[1]'s 1 Mi 256-char identity strings as HTTP bodies, drained with b9_endpoint_drain_launch. One resident window
drained with B9_DRAIN_PEEK under a callback policy (a 32-byte key), R times with the runner's bit and R times without,
alternated on the same ctx:
  - drain_ms_plain / drain_ms_runner: the median CUDA-event span around the launch's kernels (b9_stats.last_drain_kernel_ms);
    without the bit the pickle records are B9_CB_HOST and an endpoint launch runs no callback pass;
  - runner_kernel_ms: the runner's own pass (function_callback_kernel / endpoint_callback_kernel), from torch.profiler's
    CUDA activity over R launches (median);
  - d_bytes: the callback JSON bytes the pass wrote; kinds: the b9_callback_kind counts.
Prints one JSON line with the card's name and power limit read in the same run. Writes nothing.
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

KEY = b"k" * 32


def kernel_ms(dq, launch, name: str, reps: int) -> float:
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            launch()
        dq.sync()
    times = [e.device_time / 1e3 if hasattr(e, "device_time") else e.cuda_time / 1e3 for e in prof.events() if name in e.name]
    return statistics.median(times) if times else float("nan")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--runner", choices=["function", "endpoint"], required=True)
    ap.add_argument("--reps", type=int, default=9)
    a = ap.parse_args()
    from beta9_b200 import _lib as L
    from beta9_b200 import synth
    from beta9_b200.device_queue import DeviceQueue
    info = card()
    if a.runner == "function":
        b = synth.function_docs_batch(25_000)
        handler, flags, name = "json_sum", L.TF_PICKLE, "function_callback_kernel"
        launch_kw = dict(full_pickle=True)
    else:
        b = synth.strings_batch(1 << 20, 256)
        handler, flags, name = "identity", L.TF_HTTP_BODY, "endpoint_callback_kernel"
        launch_kw = dict(endpoint=True)
    with DeviceQueue(ring_bytes=1 << 31, ring_tasks=1 << 21, max_drain_tasks=1 << 21, max_result_bytes=1 << 31) as dq:
        dq.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, flags, np.uint8))
        dq.sync()
        dq.set_callback_policy(KEY)
        span = {"plain": [], "runner": []}
        for rep in range(a.reps + 1):                                      # (rep 0 warms both up)
            for mode in ("plain", "runner"):
                dq.set_callback_runners(**{a.runner: mode == "runner"})
                dq.drain_launch(handler, b.n, peek=True, **launch_kw)
                if rep:
                    span[mode].append(float(dq.stats().last_drain_kernel_ms))
        dq.set_callback_runners(**{a.runner: True})
        dq.drain_launch(handler, b.n, peek=True, **launch_kw)
        res = dq.fetch(cap_tasks=b.n, callbacks=True)
        k_ms = kernel_ms(dq, lambda: dq.drain_launch(handler, b.n, peek=True, **launch_kw), name, a.reps)
        line = {"runner": a.runner, "handler": handler, "tasks": b.n, "reps": a.reps,
                "drain_ms_plain": statistics.median(span["plain"]), "drain_ms_runner": statistics.median(span["runner"]),
                "runner_kernel_ms": k_ms, "d_bytes": int(res.cb_body_len.astype(np.int64).sum()),
                "kinds": np.bincount(res.cb_kind, minlength=4).tolist()}
        line.update(info)
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
