"""W ranks of the rebalance in ONE process on ONE GPU, through the loopback NCCL stand-in (tests/loopback_nccl).

    python tests/_loopback_rebalance_worker.py <libloopback_nccl.so> <case.pkl> <out.pkl>
    python tests/_loopback_rebalance_worker.py <libloopback_nccl.so> selftest <out.pkl>

A case is a dict: "world", "queue" (DeviceQueue keyword arguments per rank), "batches" (name -> ids, payload, offsets and
optional flags / retries / ts / exp) and "steps", run in order. Collective steps (comm_init, rebalance) run on one thread
per rank, joined with a timeout: a rank that does not come back ends the process with exit code 3, so nothing outlives
the test that started it. The results go to <out.pkl>: step tag -> one entry per rank.

Steps:
    ("push", rank, batch)                      push a batch on one rank
    ("policy", retry_mask, max_retries)        b9_set_retry_policy on every rank
    ("rebalance", tag)                         collective; per rank: rc, info, depth, depth_bytes, the loopback log of the call
    ("peek", tag, handler, opts)               per rank: a PEEK drain (opts: full_pickle, endpoint) -> its records
    ("drain", tag, handler, max_tasks)         per rank: a popping drain of at most max_tasks (None: all) -> its records
    ("drain_rank", tag, rank, handler, max_tasks)   the same on one rank
    ("expire", tag, now_ns)                    per rank: b9_expire -> the count
    ("peek_launch", handler)                   per rank: a PEEK launch whose results are left waiting
    ("fetch", tag)                             per rank: b9_drain_fetch -> records, or the error code
    ("depth", tag)                             per rank: depth, depth_bytes
    ("twin", tag, batches, retry, now_ns, [(handler, opts), ...])
                                               a fresh queue outside the communicator: the batches pushed in order, the
                                               retry policy (mask, max) or None, b9_expire(now_ns) unless None, then one
                                               PEEK drain per (handler, opts) -> records of tasks that never moved
"""
import ctypes as C
import os
import pickle
import sys
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

JOIN_S = 240


def collective(world, fn):
    """fn(rank) on one thread per rank; -> [result or exception]. A thread still running after JOIN_S ends the process."""
    out = [None] * world

    def run(r):
        try:
            out[r] = fn(r)
        except BaseException as e:        # noqa: B902 - reported to the test, which decides
            out[r] = e
    ts = [threading.Thread(target=run, args=(r,), daemon=True) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(JOIN_S)
        if t.is_alive():
            sys.stderr.write(f"a collective did not return within {JOIN_S} s\n")
            sys.stderr.flush()
            os._exit(3)
    return out


def records(r):
    return {"ids": r.task_ids.copy(), "status": r.status.copy(), "has": r.has_result.copy(), "lens": r.lengths.copy(),
            "payload": r.fifo_payload().copy(), "popped": r.n_popped}


def log_reader(lb):
    lb.lb_log_count.restype = C.c_long
    lb.lb_log_count.argtypes = [C.c_int]
    lb.lb_log_get.restype = C.c_int
    lb.lb_log_get.argtypes = [C.c_int, C.c_long, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_uint64), C.c_void_p, C.c_int]

    def entries(rank, start=0):
        out = []
        for i in range(start, lb.lb_log_count(rank)):
            op, peer, nb = C.c_int(), C.c_int(), C.c_uint64()
            words = np.zeros(64, np.uint64)
            k = lb.lb_log_get(rank, i, C.byref(op), C.byref(peer), C.byref(nb), words.ctypes.data, 64)
            out.append((op.value, peer.value, int(nb.value), words[:max(k, 0)].copy()))
        return out
    return entries


def push(q, b):
    q.push_batch(b["ids"], b["payload"], b["offsets"], timestamp_unix=b.get("ts"), expires_unix_ns=b.get("exp"),
                 retries=b.get("retries"), flags=b.get("flags"))


def run_case(lib_path, case):
    from beta9_b200 import _lib as L
    from beta9_b200.device_queue import DeviceQueue
    lb = C.CDLL(lib_path)                  # the handle libb9gpu.so dlopens: the same log
    log = log_reader(lb)
    W = case["world"]
    qs = [DeviceQueue(device=0, **case["queue"][r]) for r in range(W)]
    uid = DeviceQueue.comm_unique_id()
    res = collective(W, lambda r: qs[r].comm_init(uid, r, W))
    for e in res:
        if isinstance(e, BaseException):
            raise e
    out = {}

    def code(e):
        return e.code if isinstance(e, L.B9Error) else -1000

    for st in case["steps"]:
        op = st[0]
        if op == "push":
            push(qs[st[1]], case["batches"][st[2]])
        elif op == "policy":
            for q in qs:
                q._check(q._lib.b9_set_retry_policy(q._ctx, st[1], st[2]))
        elif op == "rebalance":
            starts = [lb.lb_log_count(r) for r in range(W)]

            def reb(r):
                try:
                    i = qs[r].rebalance()
                    return 0, (i.tasks_before, i.bytes_before, i.tasks_sent, i.bytes_sent, i.tasks_received, i.bytes_received, i.tasks_after, i.bytes_after)
                except L.B9Error as e:
                    return e.code, str(e)
            got = collective(W, reb)
            out[st[1]] = [{"rc": g[0], "info": g[1], "depth": qs[r].depth(), "depth_bytes": qs[r].depth_bytes(), "log": log(r, starts[r])}
                          if not isinstance(g, BaseException) else {"rc": -1000, "info": repr(g)} for r, g in enumerate(got)]
        elif op == "peek":
            opts = st[3] or {}
            out[st[1]] = []
            for q in qs:
                q.drain_launch(st[2], peek=True, **opts)
                out[st[1]].append(records(q.fetch()))
        elif op == "drain":
            out[st[1]] = [records(q.drain(st[2], max_tasks=st[3] if st[3] is not None else 1 << 22)) for q in qs]
        elif op == "drain_rank":
            out[st[1]] = records(qs[st[2]].drain(st[3], max_tasks=st[4] if st[4] is not None else 1 << 22))
        elif op == "expire":
            out[st[1]] = [q.expire(st[2]) for q in qs]
        elif op == "peek_launch":
            for q in qs:
                q.drain_launch(st[1], peek=True)
        elif op == "fetch":
            got = []
            for q in qs:
                try:
                    got.append(records(q.fetch()))
                except L.B9Error as e:
                    got.append(code(e))
            out[st[1]] = got
        elif op == "depth":
            out[st[1]] = [(q.depth(), q.depth_bytes()) for q in qs]
        elif op == "twin":
            _, tag, names, retry, now_ns, drains = st
            n = sum(case["batches"][b]["offsets"].shape[0] - 1 for b in names)
            nb = sum(int(case["batches"][b]["offsets"][-1]) for b in names)
            t = DeviceQueue(device=0, ring_bytes=max(1 << 16, 2 * nb), ring_tasks=max(1 << 10, 2 * n), max_drain_tasks=max(1 << 10, 2 * n),
                            max_result_bytes=max(1 << 20, 16 * nb))
            for b in names:
                push(t, case["batches"][b])
            if retry is not None:
                t._check(t._lib.b9_set_retry_policy(t._ctx, retry[0], retry[1]))
            twin = {"expired": t.expire(now_ns) if now_ns is not None else None, "drains": []}
            for h, opts in drains:
                t.drain_launch(h, peek=True, **(opts or {}))
                twin["drains"].append(records(t.fetch()))
            t.close()
            out[tag] = twin
        else:
            raise ValueError(f"unknown step {op!r}")
    for q in qs:
        q.close()
    return out


def selftest(lib_path):
    """The stand-in alone, on torch CUDA buffers: AllGather and grouped Send/Recv against numpy, and the errors."""
    import torch
    lb = C.CDLL(lib_path)

    class Uid(C.Structure):
        _fields_ = [("internal", C.c_char * 128)]
    lb.ncclGetUniqueId.argtypes = [C.POINTER(Uid)]
    lb.ncclCommInitRank.argtypes = [C.POINTER(C.c_void_p), C.c_int, Uid, C.c_int]
    lb.ncclAllGather.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
    lb.ncclSend.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lb.ncclRecv.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lb.ncclCommDestroy.argtypes = [C.c_void_p]
    lb.ncclGetErrorString.restype = C.c_char_p
    log = log_reader(lb)
    out = {}
    W = 3
    uid = Uid()
    assert lb.ncclGetUniqueId(C.byref(uid)) == 0
    comms = [C.c_void_p() for _ in range(W)]

    def init(r):
        torch.cuda.set_device(0)
        torch.zeros(1, device="cuda")
        return lb.ncclCommInitRank(C.byref(comms[r]), W, uid, r)
    assert collective(W, init) == [0] * W
    rng = np.random.default_rng(5)
    # AllGather of uint64 words (count 7: logged) and of bytes (count 1000)
    for count, dt, np_t, tt in ((7, 5, np.uint64, torch.int64), (1000, 1, np.uint8, torch.uint8)):
        src = [rng.integers(0, 255 if np_t is np.uint8 else 1 << 62, count).astype(np_t) for _ in range(W)]

        def ag(r):
            torch.cuda.set_device(0)
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                a = torch.from_numpy(src[r].view(np.int64) if np_t is np.uint64 else src[r]).to("cuda", non_blocking=True)
                b = torch.full((W * count,), 7, dtype=tt, device="cuda")
                rc = lb.ncclAllGather(a.data_ptr(), b.data_ptr(), count, dt, comms[r], s.cuda_stream)
                got = b.cpu().numpy()
            return rc, got.view(np_t) if np_t is np.uint64 else got
        out[f"allgather_{count}"] = (src, collective(W, ag))
    # grouped all-to-all of uneven byte counts, two messages per ordered pair
    sizes = {(s, d, k): int(rng.integers(0, 5000)) for s in range(W) for d in range(W) for k in range(2) if s != d}
    data = {key: rng.integers(0, 256, n).astype(np.uint8) for key, n in sizes.items()}

    def a2a(r):
        torch.cuda.set_device(0)
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            tx = {key: torch.from_numpy(v).to("cuda") for key, v in data.items() if key[0] == r}
            rx = {key: torch.zeros(sizes[key] + 1, dtype=torch.uint8, device="cuda") for key in sizes if key[1] == r}
            lb.ncclGroupStart()
            for d in range(W):
                if d == r:
                    continue
                for k in range(2):
                    lb.ncclSend(tx[(r, d, k)].data_ptr(), sizes[(r, d, k)], 1, d, comms[r], s.cuda_stream)
                    lb.ncclRecv(rx[(d, r, k)].data_ptr(), sizes[(d, r, k)], 1, d, comms[r], s.cuda_stream)
            rc = lb.ncclGroupEnd()
            return rc, {key: v.cpu().numpy() for key, v in rx.items()}
    out["a2a"] = (data, collective(W, a2a))
    # a Send and a Recv whose byte counts differ: both sides get an error that says so
    def mismatch(r):
        torch.cuda.set_device(0)
        buf = torch.zeros(64, dtype=torch.uint8, device="cuda")
        lb.ncclGroupStart()
        if r == 0:
            lb.ncclSend(buf.data_ptr(), 16, 1, 1, comms[r], None)
        elif r == 1:
            lb.ncclRecv(buf.data_ptr(), 32, 1, 0, comms[r], None)
        rc = lb.ncclGroupEnd()
        return rc, (lb.ncclGetErrorString(rc) or b"").decode()
    out["mismatch"] = collective(W, mismatch)
    out["log"] = [log(r) for r in range(W)]
    # an unmatched Send: an error after the timeout (LB_NCCL_TIMEOUT_S), not a hang
    buf = torch.zeros(16, dtype=torch.uint8, device="cuda")
    rc = lb.ncclSend(buf.data_ptr(), 16, 1, 2, comms[0], None)
    out["unmatched"] = (rc, (lb.ncclGetErrorString(rc) or b"").decode())
    rc2 = lb.ncclAllGather(buf.data_ptr(), buf.data_ptr(), 1, 1, comms[0], None)
    out["after_break"] = (rc2, (lb.ncclGetErrorString(rc2) or b"").decode())
    for c in comms:
        lb.ncclCommDestroy(c)
    return out


def main():
    lib_path, what, out_path = sys.argv[1], sys.argv[2], sys.argv[3]
    os.environ["B9_NCCL_LIB"] = lib_path               # before libb9gpu.so loads NCCL
    os.environ.setdefault("B9_COMM_WARMUP_BYTES", "4096")
    if what == "selftest":
        out = selftest(lib_path)
    else:
        with open(what, "rb") as f:
            case = pickle.load(f)
        out = run_case(lib_path, case)
    with open(out_path + ".tmp", "wb") as f:
        pickle.dump(out, f)
    os.replace(out_path + ".tmp", out_path)


if __name__ == "__main__":
    main()
