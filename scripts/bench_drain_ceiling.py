"""How close configs[1]'s identity drain comes to what a plain device copy reaches on the same card.

    python scripts/bench_drain_ceiling.py [--steps K] [--warmup W] [--rounds R] [--kernel-copies-ids]

In one process on one GPU, alternated R times:
  drain   configs[1] (1 M x 256-char identity tasks, 1 % escapes) timed as bench.py times it: K B9_DRAIN_PEEK launches
          enqueued back to back, CUDA events from the first one's start to the last one's end
  copy    a device-to-device cudaMemcpyAsync (torch's copy_ of a contiguous uint8 tensor) whose read + write volume is
          the drain's real bytes per step, once for the record layout that copies each record's id through the kernel
          (62 B of slot and record words per task) and once for the one that leaves ids in the ring (30 B)
The drain's real bytes per step are its payload bytes in, its result bytes out and its slot and record words per task
(32 B fewer per task when ids stay in the ring; --kernel-copies-ids accounts a library built before that change, loaded
with B9GPU_LIB). Prints one JSON line: ms per step, GB/s and their ratio, with the card's name and power limit read in
the same run. Fails without a GPU."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SLOT_WORDS = 8 + 8           # payload offset + header word per task (ring slot words the drain reads)
RECORD_WORDS = 8 + 4 + 1 + 1  # offset, length, status, has_result per record
ID_BYTES = 16


def gpu_info(device: int) -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                          "-i", str(device)], capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
    return {"name": out[0], "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--tasks", type=int, default=1_000_000, help="tasks per step (configs[1] on one GPU: 1 M)")
    ap.add_argument("--chars", type=int, default=256)
    ap.add_argument("--kernel-copies-ids", action="store_true", help="the loaded library copies every record's id in the kernel")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_drain_ceiling.py: no CUDA device")
    torch.cuda.set_device(0)
    from beta9_b200 import synth
    from beta9_b200.device_queue import DeviceQueue

    b = synth.strings_batch(a.tasks, a.chars, adversarial_frac=0.01, seed=synth.SEED)
    n, in_bytes = b.n, int(b.payload.size)
    dq = DeviceQueue(device=0, ring_bytes=max(1 << 30, 4 * in_bytes), ring_tasks=max(1 << 21, 4 * n),
                     max_drain_tasks=max(1 << 21, 2 * n), max_result_bytes=max(1 << 30, 3 * in_bytes))
    dq.push_batch(b.task_ids, b.payload, b.offsets)
    for _ in range(a.warmup):
        dq.drain_launch("identity", n, peek=True)
    out_bytes = int(dq.stats().last_drain_out_bytes)

    def drain_ms() -> float:
        torch.cuda.synchronize()
        for _ in range(a.steps):
            dq.drain_launch("identity", n, peek=True, wait=False)
        dq.sync()
        return float(dq.stats().last_drain_kernel_ms) / a.steps

    words = {"ids_copied": SLOT_WORDS + RECORD_WORDS + 2 * ID_BYTES, "ids_in_ring": SLOT_WORDS + RECORD_WORDS}
    volume = {k: in_bytes + out_bytes + w * n for k, w in words.items()}          # read + write bytes per step
    bufs = {k: (torch.empty(v // 2, dtype=torch.uint8, device="cuda"), torch.empty(v // 2, dtype=torch.uint8, device="cuda"))
            for k, v in volume.items()}
    for src, _ in bufs.values():
        src.fill_(1)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def copy_ms(k: str) -> float:
        src, dst = bufs[k]
        for _ in range(a.warmup):
            dst.copy_(src)
        ev0.record()
        for _ in range(a.steps):
            dst.copy_(src)
        ev1.record()
        ev1.synchronize()
        return ev0.elapsed_time(ev1) / a.steps

    runs = {"drain": [], "copy_ids_copied": [], "copy_ids_in_ring": []}
    for _ in range(a.rounds):
        runs["drain"].append(drain_ms())
        for k in words:
            runs["copy_" + k].append(copy_ms(k))
    drain_volume = volume["ids_copied" if a.kernel_copies_ids else "ids_in_ring"]
    med = {k: statistics.median(v) for k, v in runs.items()}

    def gbs(nbytes: int, ms: float) -> float:
        return nbytes / (ms * 1e-3) / 1e9

    line = {
        "workload": f"configs[1]: {n} x {a.chars}-char identity tasks, 1% escapes; {a.steps} steps x {a.rounds} rounds",
        "gpu": gpu_info(0),
        "bytes_per_task": {"payload_in": in_bytes / n, "result_out": out_bytes / n, **{k: v / n for k, v in volume.items()}},
        "kernel_copies_ids": a.kernel_copies_ids,
        "drain": {"ms_per_step": med["drain"], "runs_ms": runs["drain"], "bytes_per_step": drain_volume,
                  "gb_per_s": gbs(drain_volume, med["drain"])},
        "copy": {k: {"ms": med["copy_" + k], "runs_ms": runs["copy_" + k], "bytes": volume[k], "gb_per_s": gbs(volume[k], med["copy_" + k])}
                 for k in words},
    }
    line["drain_over_copy"] = line["drain"]["gb_per_s"] / line["copy"]["ids_copied" if a.kernel_copies_ids else "ids_in_ring"]["gb_per_s"]
    print(json.dumps(line))
    dq.close()


if __name__ == "__main__":
    main()
