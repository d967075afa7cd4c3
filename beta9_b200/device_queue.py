"""Python face of one b9_ctx: a device-resident task queue for one GPU.

Mirrors `taskQueueClient` (pkg/abstractions/taskqueue/client.go:29-106: Push / Pop / QueueLength)
batch-wise: `push_batch` = n x Push, `drain` = up to n x (Pop + runner loop + Complete hand-off).
All buffers are numpy arrays; results come back packed (see `DrainResult`).
"""
from __future__ import annotations

import binascii
import ctypes as C
import os
import uuid
from dataclasses import dataclass
from typing import Iterable, List, Optional, Tuple, Union

import numpy as np

from . import _lib as L

HANDLERS = {"identity": L.H_IDENTITY, "echo": L.H_IDENTITY, "crc32": L.H_CRC32,
            "vadd_f32": L.H_VADD_F32, "json_sum": L.H_JSON_SUM}
STATUS_NAMES = {L.ST_COMPLETE: "COMPLETE", L.ST_ERROR: "ERROR", L.ST_RETRY: "RETRY",
                L.ST_REJECTED: "REJECTED", L.ST_UNSUPPORTED: "UNSUPPORTED", L.ST_RETRY_LIMIT: "RETRY_LIMIT"}
# every exception class a device handler can raise, and its B9_EXC_* bit (include/b9gpu.h)
EXC_BITS = {TypeError: L.EXC_TYPE_ERROR, AttributeError: L.EXC_ATTRIBUTE_ERROR, UnicodeEncodeError: L.EXC_UNICODE_ENCODE,
            KeyError: L.EXC_KEY_ERROR, ValueError: L.EXC_VALUE_ERROR, binascii.Error: L.EXC_BINASCII_ERROR}


def retry_mask(retry_for: Optional[Iterable[type]]) -> int:
    """The B9_EXC_* bits of a `retry_for` list. The runner retries on `type(e) is err` (retry_on_errors, an exact match),
    so classes map by identity: a subclass or a class outside EXC_BITS is never what a device handler raises, and adds
    nothing."""
    m = 0
    for err in retry_for or ():
        for cls, bit in EXC_BITS.items():
            if err is cls:
                m |= bit
    return m


@dataclass
class DrainResult:
    task_ids: np.ndarray     # uint8 [n,16]
    status: np.ndarray       # uint8 [n]
    has_result: np.ndarray   # uint8 [n]
    offsets: np.ndarray      # uint64 [n]   start of record i's bytes in `payload`
    lengths: np.ndarray      # uint32 [n]
    payload: np.ndarray      # uint8 [n_bytes]  byte order = tile completion order (16-byte padded ranges), use offsets
    n_popped: int
    task_duration: float = 0.0   # seconds charged to every task of the drain (TaskQueueCompleteRequest.task_duration)
    # with callbacks=True (b9_drain_fetch_callbacks): the runner's callback per record
    cb_kind: Optional[np.ndarray] = None     # uint8 [n]     CB_NONE / CB_POST / CB_UNSENDABLE / CB_HOST
    cb_digest: Optional[np.ndarray] = None   # uint8 [n,32]  raw HMAC-SHA256 of a CB_POST record under a key, else zero
    cb_timestamp: int = 0                    # the Unix seconds every digest signs (0: no key)
    # under set_callback_runners (b9_drain_fetch_callback_requests): each record's callback JSON D and own URL in `payload`
    cb_body_off: Optional[np.ndarray] = None  # uint64 [n]
    cb_body_len: Optional[np.ndarray] = None  # uint32 [n]   0: D is {}
    cb_url_off: Optional[np.ndarray] = None   # uint64 [n]
    cb_url_len: Optional[np.ndarray] = None   # uint32 [n]   0: the stub's URL

    @property
    def n(self) -> int:
        return int(self.status.shape[0])

    def result(self, i: int) -> Optional[bytes]:
        if not self.has_result[i]:
            return None
        o = int(self.offsets[i])
        return self.payload[o:o + int(self.lengths[i])].tobytes()

    def fifo_payload(self) -> np.ndarray:
        """The result bytes re-laid in record order (what `offsets[n+1]`-style consumers expect)."""
        if self.n == 0:
            return np.empty(0, np.uint8)
        ln = self.lengths.astype(np.int64)
        ends = np.cumsum(ln)
        idx = np.arange(int(ends[-1]), dtype=np.int64)
        rec = np.repeat(np.arange(self.n, dtype=np.int64), ln)
        src = self.offsets.astype(np.int64)[rec] + (idx - (ends - ln)[rec])
        return self.payload[src]

    def callback_body(self, i: int) -> bytes:
        """The bytes the runner signs and posts for record i: {"data": R}, or {"data": {}} without result bytes; under
        callback runners {"data": D}, D being the callback JSON the device wrote (R itself for task-queue records)."""
        if self.cb_body_len is not None:
            n = int(self.cb_body_len[i])
            o = int(self.cb_body_off[i])
            return b'{"data": ' + (self.payload[o:o + n].tobytes() if n else b"{}") + b"}"
        r = self.result(i)
        return b'{"data": ' + (r if r is not None else b"{}") + b"}"

    def callback_url(self, i: int) -> Optional[str]:
        """The task's own callback URL (a function task's callback_url kwarg), or None: the stub's URL."""
        if self.cb_url_len is None or not int(self.cb_url_len[i]):
            return None
        o = int(self.cb_url_off[i])
        return self.payload[o:o + int(self.cb_url_len[i])].tobytes().decode("utf-8")

    def callback_headers(self, i: int, status: Optional[str] = None) -> dict:
        """send_callback's headers for record i (status: the runner's TaskStatus, by default the record's)."""
        sig = self.cb_digest[i].tobytes().hex() if self.cb_timestamp else ""
        return {"X-Task-ID": str(uuid.UUID(bytes=self.task_ids[i].tobytes())),
                "X-Task-Status": status or STATUS_NAMES[int(self.status[i])],
                "X-Task-Signature": sig, "X-Task-Timestamp": str(self.cb_timestamp)}

    def records(self) -> List[Tuple[bytes, str, Optional[bytes]]]:
        return [(self.task_ids[i].tobytes(), STATUS_NAMES[int(self.status[i])], self.result(i)) for i in range(self.n)]


class PinnedBuffer:
    """Page-locked host memory from b9_host_alloc, viewed as a numpy array."""

    def __init__(self, q: "DeviceQueue", nbytes: int):
        self._q = q
        self.nbytes = int(nbytes)
        self.ptr = q._lib.b9_host_alloc(q._ctx, self.nbytes)
        if not self.ptr:
            raise L.B9Error(L.B9_ENOMEM, L.last_error())
        self.array = np.ctypeslib.as_array((C.c_uint8 * max(1, self.nbytes)).from_address(self.ptr))[:self.nbytes]

    def view(self, dtype, count: int, offset: int = 0) -> np.ndarray:
        return self.array[offset:offset + count * np.dtype(dtype).itemsize].view(dtype)

    def free(self) -> None:
        if self.ptr:
            self.array = None
            self._q._lib.b9_host_free(self._q._ctx, self.ptr)
            self.ptr = None


class DeviceQueue:
    def __init__(self, device: int = 0, ring_bytes: int = 0, ring_tasks: int = 0, max_drain_tasks: int = 0,
                 max_result_bytes: int = 0, max_task_bytes: int = 0):
        self._lib = L.load()
        o = L.Opts(C.sizeof(L.Opts), device, ring_bytes, ring_tasks, max_drain_tasks, max_result_bytes, max_task_bytes, 0)
        ctx = C.c_void_p()
        rc = self._lib.b9_ctx_create(C.byref(o), C.byref(ctx))
        if rc != L.B9_OK:
            raise L.B9Error(rc, L.last_error())
        self._ctx = ctx
        self.device = device
        self._res_bufs = None
        self._user_handlers = {}                   # name -> id of the handlers load_handler loaded into this context

    def close(self) -> None:
        if getattr(self, "_ctx", None):
            self._lib.b9_ctx_destroy(self._ctx)
            self._ctx = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _check(self, rc: int) -> int:
        if rc < 0:
            raise L.B9Error(int(rc), L.last_error(self._ctx))
        return int(rc)

    # ---- producer side (client.go:29-41 Push, batch-wise)
    def push_batch(self, task_ids: np.ndarray, payload: np.ndarray, offsets: np.ndarray,
                   timestamp_unix: Optional[np.ndarray] = None, expires_unix_ns: Optional[np.ndarray] = None,
                   retries: Optional[np.ndarray] = None, flags: Optional[np.ndarray] = None) -> None:
        ids = np.ascontiguousarray(task_ids, dtype=np.uint8)
        pl = np.ascontiguousarray(payload, dtype=np.uint8)
        off = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = off.shape[0] - 1
        assert ids.size == n * 16, "task_ids must be n x 16 bytes"
        keep = []

        def ptr(a, dt):
            if a is None:
                return None
            a = np.ascontiguousarray(a, dtype=dt)
            assert a.shape[0] == n
            keep.append(a)
            return a.ctypes.data
        meta = L.PushMeta(ptr(timestamp_unix, np.int64), ptr(expires_unix_ns, np.int64), ptr(retries, np.uint8), ptr(flags, np.uint8))
        self._check(self._lib.b9_batch_push(self._ctx, ids.ctypes.data, pl.ctypes.data if pl.size else ids.ctypes.data,
                                            off.ctypes.data, n, C.byref(meta)))

    def push_scattered(self, task_ids: np.ndarray, pointers: np.ndarray, lengths: np.ndarray) -> None:
        """b9_batch_push_v: `pointers` uint64[n] host addresses of the payloads (anywhere in pageable memory),
        `lengths` uint32[n]. The library gathers them into its page-locked arena (the pack step) and pushes that."""
        ids = np.ascontiguousarray(task_ids, dtype=np.uint8)
        ptrs = np.ascontiguousarray(pointers, dtype=np.uint64)
        lens = np.ascontiguousarray(lengths, dtype=np.uint32)
        n = lens.shape[0]
        assert ids.size == n * 16 and ptrs.shape[0] == n
        self._check(self._lib.b9_batch_push_v(self._ctx, ids.ctypes.data, ptrs.ctypes.data, lens.ctypes.data, n, None))

    def submit(self, task_id: bytes, payload: bytes, flags: int = 0) -> None:
        """b9_submit: one task (16 raw id bytes + payload) from any thread; batched under the hood, `flush()` pushes."""
        self._check(self._lib.b9_submit(self._ctx, task_id, payload, len(payload), flags))

    def flush(self) -> int:
        return self._check(self._lib.b9_flush(self._ctx))

    def buffered(self) -> int:
        return int(self._lib.b9_buffered(self._ctx))

    def depth(self) -> int:                       # client.go:99-106 QueueLength / task_redis.go:112-119 TasksInFlight
        return int(self._lib.b9_depth(self._ctx))

    def running(self) -> int:                     # task_redis.go:58 TasksClaimed / client.go:109 TasksRunning
        return int(self._lib.b9_running(self._ctx))

    def depth_bytes(self) -> int:
        return int(self._lib.b9_depth_bytes(self._ctx))

    def expire(self, now_unix_ns: int) -> int:    # dispatch.go:173-230 monitor, unclaimed branch
        return self._check(self._lib.b9_expire(self._ctx, now_unix_ns))

    def cancel(self, task_ids: np.ndarray) -> Tuple[int, np.ndarray]:   # api/v1/task.go:333-398 StopTasks
        """b9_cancel: marks the pending, unclaimed tasks with these ids (uint8 [n,16]) cancelled. Returns (slots marked,
        uint8 [n] outcome: an OR of CANCEL_MARKED / CANCEL_ALREADY / CANCEL_CLAIMED, 0 = no such pending task)."""
        ids = np.ascontiguousarray(task_ids, dtype=np.uint8).reshape(-1, 16)
        n = ids.shape[0]
        outcome = np.zeros(max(n, 1), np.uint8)
        marked = self._check(self._lib.b9_cancel(self._ctx, ids.ctypes.data if n else None, n, outcome.ctypes.data))
        return marked, outcome[:n]

    def set_callback_policy(self, signing_key: Optional[bytes]) -> None:
        """b9_set_callback_policy: the stub has a callback URL and its workspace signs with `signing_key` (b"": the gateway
        without a key; the runner then posts unsigned). None turns the callback pass off. Drains launched after it run
        the pass; fetch them with callbacks=True."""
        if signing_key is None:
            self._check(self._lib.b9_set_callback_policy(self._ctx, 0, None, 0))
        else:
            key = bytes(signing_key)
            self._check(self._lib.b9_set_callback_policy(self._ctx, 1, key if key else None, len(key)))

    def set_callback_runners(self, function: bool = False, endpoint: bool = False) -> None:
        """b9_set_callback_runners: under the callback policy, also settle the function runner's callbacks (pickle tasks of
        full_pickle=True drains) and the endpoint runner's (endpoint=True drains) on the device. fetch(callbacks=True) then
        carries each record's callback JSON and URL (callback_body, callback_url)."""
        runners = (L.CB_RUNNER_FUNCTION if function else 0) | (L.CB_RUNNER_ENDPOINT if endpoint else 0)
        self._check(self._lib.b9_set_callback_runners(self._ctx, runners))
        self._cb_runners = runners

    def set_retry_policy(self, retry_for: Optional[Iterable[type]], max_retries: int) -> None:
        """b9_set_retry_policy: the stub's `retry_for` classes and TaskPolicy.MaxRetries. A task whose handler raised one of
        them comes back RETRY (and is pushed again, retries + 1, when its drain is fetched) or, once its retries reached
        max_retries, RETRY_LIMIT. An empty `retry_for` restores the answers without a policy. max_retries is at most 255
        (a task's retries are one byte); a larger value raises B9Error (B9_EINVAL)."""
        self._check(self._lib.b9_set_retry_policy(self._ctx, retry_mask(retry_for), max(0, int(max_retries))))

    # ---- user handlers
    def load_handler(self, image: Union[bytes, str, os.PathLike], name: str) -> int:
        """b9_handler_load: loads the B9_HANDLER `name` of an sm_90a cubin or fatbin (its bytes, or a path to it) compiled
        against include/b9gpu_handler.cuh (build.compile_handlers). Returns its id (H_USER_BASE + k); drains then take
        `name` or the id wherever they take a built-in handler's name."""
        if not isinstance(image, (bytes, bytearray, memoryview)):
            with open(image, "rb") as f:
                image = f.read()
        data = bytes(image)
        hid = C.c_int32(0)
        self._check(self._lib.b9_handler_load(self._ctx, data, len(data), name.encode(), C.byref(hid)))
        self._user_handlers[name] = int(hid.value)
        return int(hid.value)

    def handler_id(self, handler: Union[str, int]) -> int:
        """The id of a built-in handler's name, of a name load_handler loaded, or an id as it is."""
        if isinstance(handler, int):
            return handler
        if handler in self._user_handlers:
            return self._user_handlers[handler]
        return HANDLERS[handler]

    # ---- consumer side
    def drain(self, handler: Union[str, int], max_tasks: int = 1 << 22, cap_bytes: Optional[int] = None, full_pickle: bool = False,
              endpoint: bool = False, callbacks: bool = False) -> DrainResult:
        """full_pickle=True (B9_DRAIN_PICKLE_FULL): pickle-framed tasks of every handler over plain values (include/b9gpu.h).
        endpoint=True (b9_endpoint_drain_launch): B9_TF_HTTP_BODY tasks answered with the endpoint runner's response bodies.
        callbacks=True (b9_drain_fetch_callbacks, under set_callback_policy): the result carries each record's callback."""
        n = self._launch(self.handler_id(handler), max_tasks, L.DRAIN_PICKLE_FULL if full_pickle else 0, endpoint)
        return self._fetch(n, cap_bytes, callbacks)

    def drain_launch(self, handler: Union[str, int], max_tasks: int = 1 << 22, peek: bool = False, wait: bool = True, full_pickle: bool = False,
                     endpoint: bool = False) -> int:
        """wait=False (B9_DRAIN_ASYNC): returns once the kernels are enqueued; `sync()` or `fetch()` completes it."""
        flags = (1 if peek else 0) | (0 if wait else 2) | (L.DRAIN_PICKLE_FULL if full_pickle else 0)
        return self._launch(self.handler_id(handler), max_tasks, flags, endpoint)

    def _launch(self, h: int, max_tasks: int, flags: int, endpoint: bool) -> int:
        if not endpoint:
            return self._check(self._lib.b9_drain_launch(self._ctx, h, max_tasks, flags))
        if flags & L.DRAIN_PICKLE_FULL:
            raise ValueError("endpoint=True answers HTTP bodies only: it does not combine with full_pickle=True")
        return self._check(self._lib.b9_endpoint_drain_launch(self._ctx, h, max_tasks, flags))

    def fetch(self, cap_bytes: Optional[int] = None, callbacks: bool = False, cap_tasks: Optional[int] = None) -> DrainResult:
        self.sync()                                  # completes a wait=False launch: its byte count sizes the buffers below
        st = self.stats()
        return self._fetch(cap_tasks, cap_bytes if cap_bytes is not None else int(st.last_drain_out_bytes), callbacks)

    def _fetch(self, n: Optional[int], cap_bytes: Optional[int], callbacks: bool = False) -> DrainResult:
        st = self.stats()
        if cap_bytes is None:
            cap_bytes = int(st.last_drain_out_bytes)
        if n is None:
            n = int(st.last_drain_tiles) * 128      # an upper bound for either kernel generation
        ids = np.empty((max(n, 1), 16), np.uint8)
        status = np.empty(max(n, 1), np.uint8)
        has = np.empty(max(n, 1), np.uint8)
        off = np.zeros(max(n, 1), np.uint64)
        ln = np.zeros(max(n, 1), np.uint32)
        pl = np.empty(max(cap_bytes, 1), np.uint8)
        r = L.Results(ids.ctypes.data, status.ctypes.data, has.ctypes.data, off.ctypes.data, ln.ctypes.data, pl.ctypes.data,
                      max(n, 1), max(cap_bytes, 1), 0, 0, 0, 0, 0.0, 0)
        if not callbacks:
            got = self._check(self._lib.b9_drain_fetch(self._ctx, C.byref(r)))
            return DrainResult(ids[:got], status[:got], has[:got], off[:got], ln[:got], pl[:int(r.n_bytes)], int(r.n_popped), float(r.task_duration))
        kind = np.empty(max(n, 1), np.uint8)
        digest = np.empty((max(n, 1), 32), np.uint8)
        cb = L.Callbacks(kind.ctypes.data, digest.ctypes.data, max(n, 1), 0)
        if not getattr(self, "_cb_runners", 0):
            got = self._check(self._lib.b9_drain_fetch_callbacks(self._ctx, C.byref(r), C.byref(cb)))
            return DrainResult(ids[:got], status[:got], has[:got], off[:got], ln[:got], pl[:int(r.n_bytes)], int(r.n_popped), float(r.task_duration),
                               kind[:got], digest[:got], int(cb.timestamp))
        b_off = np.zeros(max(n, 1), np.uint64)
        b_len = np.zeros(max(n, 1), np.uint32)
        u_off = np.zeros(max(n, 1), np.uint64)
        u_len = np.zeros(max(n, 1), np.uint32)
        rq = L.CallbackRequests(b_off.ctypes.data, b_len.ctypes.data, u_off.ctypes.data, u_len.ctypes.data, max(n, 1))
        got = self._check(self._lib.b9_drain_fetch_callback_requests(self._ctx, C.byref(r), C.byref(cb), C.byref(rq)))
        return DrainResult(ids[:got], status[:got], has[:got], off[:got], ln[:got], pl[:int(r.n_bytes)], int(r.n_popped), float(r.task_duration),
                           kind[:got], digest[:got], int(cb.timestamp), b_off[:got], b_len[:got], u_off[:got], u_len[:got])

    def drain_object(self, handler: Union[str, int], max_tasks: int = 1 << 22, endpoint: bool = False) -> np.ndarray:
        """One drain whose records land as ONE result-sink object (b9_drain_fetch_object): header + index + blob."""
        self._launch(self.handler_id(handler), max_tasks, 0, endpoint)
        need = C.c_uint64(0)
        probe = np.zeros(128, np.uint8)
        rc = self._lib.b9_drain_fetch_object(self._ctx, probe.ctypes.data, 0, C.byref(need))      # B9_ENOSPC: tells the size, consumes nothing
        if rc != L.B9_ENOSPC:
            self._check(rc)
        obj = np.empty(int(need.value), np.uint8)
        self._check(self._lib.b9_drain_fetch_object(self._ctx, obj.ctypes.data, obj.size, C.byref(need)))
        return obj

    def drain_into(self, handler: Union[str, int], max_tasks: int, res: "L.Results") -> int:
        """b9_drain straight into caller-owned (ideally pinned) buffers described by `res`."""
        return self._check(self._lib.b9_drain(self._ctx, self.handler_id(handler), max_tasks, C.byref(res)))

    def wire_encode(self, workspace_name: str, stub_id: str, max_tasks: int = 1 << 22, executor: str = "taskqueue",
                    max_retries: int = 3, timeout: int = 3600, ttl: int = 7200, full: bool = False) -> DrainResult:
        """TaskMessage.Encode (pkg/types/task.go:79-90) of the pending tasks, on the device; they stay pending.
        full=True: b9_wire_encode_full (floats, unsorted / duplicate keys, HTTP bodies; include/b9gpu.h)."""
        env = L.WireEnv(workspace_name.encode(), stub_id.encode(), executor.encode(), max_retries, timeout, ttl)
        fn = self._lib.b9_wire_encode_full if full else self._lib.b9_wire_encode
        n = self._check(fn(self._ctx, C.byref(env), max_tasks))
        return self._fetch(n, None)

    # ---- multi-GPU (one DeviceQueue per rank / GPU)
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = (C.c_uint8 * 128)()
        rc = L.load().b9_comm_unique_id(buf)
        if rc != 0:
            raise L.B9Error(rc, L.last_error())
        return bytes(buf)

    def comm_init(self, unique_id: bytes, rank: int, world: int) -> None:
        buf = (C.c_uint8 * 128).from_buffer_copy(unique_id)
        self._check(self._lib.b9_comm_init(self._ctx, buf, rank, world))

    def rebalance(self) -> "L.RebalanceInfo":
        """Collective: byte-quantile rebalance of the pending ring over the communicator (NCCL all-to-all)."""
        info = L.RebalanceInfo()
        self._check(self._lib.b9_rebalance(self._ctx, C.byref(info)))
        return info

    def stats(self) -> "L.Stats":
        s = L.Stats()
        self._check(self._lib.b9_stats_get(self._ctx, C.byref(s)))
        return s

    def sync(self) -> None:
        self._check(self._lib.b9_sync(self._ctx))

    def pinned(self, nbytes: int) -> PinnedBuffer:
        return PinnedBuffer(self, nbytes)


def rebalance_plan(world: int, rank: int, counts, nbytes, prefix) -> Tuple[np.ndarray, np.ndarray]:
    """b9_rebalance_plan: local FIFO range [lo[d], hi[d]) destined for every rank d (pure host arithmetic)."""
    counts = np.ascontiguousarray(counts, np.uint64); nbytes = np.ascontiguousarray(nbytes, np.uint64)
    prefix = np.ascontiguousarray(prefix, np.uint64)
    lo = np.zeros(world, np.uint64); hi = np.zeros(world, np.uint64)
    rc = L.load().b9_rebalance_plan(world, rank, counts.ctypes.data, nbytes.ctypes.data, prefix.ctypes.data,
                                    prefix.shape[0] - 1, lo.ctypes.data, hi.ctypes.data)
    if rc != 0:
        raise L.B9Error(rc, L.last_error())
    return lo, hi


def task_queue_scale(queue_length: int, tasks_per_container: int, max_containers: int, max_replicas: int) -> Tuple[int, bool]:
    """taskQueueScaleFunc (pkg/abstractions/taskqueue/autoscaler.go:53-79) via the C ABI."""
    v = C.c_int(0)
    d = L.load().b9_task_queue_scale(queue_length, tasks_per_container, max_containers, max_replicas, C.byref(v))
    return int(d), bool(v.value)
