"""A plain Python model of one device queue (one b9_ctx), for checking random sequences of calls against the library.

It keeps what the host keeps (the pending FIFO, the claimed window of an outstanding launch, the policies, the push
segments) and answers every call the way the library must. The answers themselves are never restated here: statuses
and result bytes come from tests/retry_oracle.py (oracle/pyoracle/loop.py's loop with the stub's retry policy),
callback kinds and digests from oracle/pyoracle/callback.py, endpoint bodies from oracle/pyoracle/endpoint.py and
pickle-framed answers from oracle/pyoracle/funcloop.py. What the model adds are the queue's rules, each next to the
place that defines it.

`OpGen` draws a deterministic sequence of operations for a seed; `apply` plays one logged operation on a model, so a
logged sequence replays exactly (tests/test_gpu_queue_model.py plays the same operations on a device queue)."""
from __future__ import annotations

import binascii
import hashlib
import hmac
import json
import random
import uuid
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

from oracle.pyoracle import callback as CB
from oracle.pyoracle import endpoint as EP
from oracle.pyoracle import funcloop
from oracle.pyoracle.gojson import GoJSONError, go_unmarshal_task_payload
from oracle.pyoracle.httpserialize import InvalidRequestPayload, serialize_http_payload
from oracle.pyoracle.loop import run_task_loop, sdk_put_payload
from tests.retry_oracle import run_retry_loop

# include/b9gpu.h
TF_CANCELLED, TF_HTTP_BODY, TF_PICKLE, TF_TASK_MSG = 0x01, 0x02, 0x04, 0x08
MARKED, ALREADY, CLAIMED = 0x01, 0x02, 0x04
HANDLERS = ["identity", "crc32", "vadd_f32", "json_sum"]
# every class a device handler raises (beta9_b200/device_queue.py EXC_BITS)
RETRY_CLASSES = [TypeError, AttributeError, UnicodeEncodeError, KeyError, ValueError, binascii.Error]
SEG_ALIGN = 256                       # B9_SEG_ALIGN (ring_place.h)
RECORD_BYTES = 16 + 1 + 1 + 8 + 4     # what a fetch reads back per record besides its bytes: id, status, has_result, offset, length


def seg_span(nbytes: int) -> int:
    """b9_seg_span (ring_place.h): the ring bytes a push segment of `nbytes` occupies."""
    return (nbytes + SEG_ALIGN - 1) // SEG_ALIGN * SEG_ALIGN


def pow2_ceil(v: int) -> int:
    p = 1
    while p < v:
        p <<= 1
    return p


class ModelError(Exception):
    """A call the library must refuse: `code` is the B9_E* value it returns (nothing changes)."""

    def __init__(self, code: int, what: str):
        super().__init__(f"{code}: {what}")
        self.code = code


B9_EINVAL, B9_ENOSPC = -22, -28


@dataclass
class Task:
    id: bytes
    payload: bytes
    flags: int = 0
    retries: int = 0
    expires: int = 0                        # Unix ns; 0 = never
    ts: Tuple[int, int] = (0, 0)            # its slot's timestamp lies in [lo, hi] (a push's own; a re-push: the commit's clock)
    repushed: bool = False


@dataclass
class Record:
    id: bytes
    status: str
    result: Optional[bytes]
    kind: int                               # b9_callback_kind under a callback policy


@dataclass
class Window:
    """The launch whose records wait for a fetch."""
    n: int                                  # window tasks (popped at the commit)
    peek: bool
    endpoint: bool
    records: List[Record]
    retry: List[Task]                       # the tasks of its RETRY records, in record order
    callbacks: bool                         # the launch ran the callback pass
    key: bytes                              # its signing key (b"": unsigned)


class QueueModel:
    def __init__(self, ring_bytes: int, ring_tasks: int, max_drain_tasks: int = 0):
        # b9_ctx_create's rounding (b9gpu.cu)
        self.ring_bytes = pow2_ceil(ring_bytes)
        self.ring_tasks = pow2_ceil(ring_tasks)
        self.max_drain_tasks = min(max_drain_tasks or (2 << 20), self.ring_tasks, (1 << 24) - 1)
        self.pending: List[Task] = []
        self.segs: List[List[int]] = []      # push segments in FIFO order: [tasks not yet popped, ring bytes held]
        self.window: Optional[Window] = None
        self.retry_for: Tuple[type, ...] = ()
        self.max_retries = 0
        self.cb_key: Optional[bytes] = None  # None: no callback policy
        self.tasks_drained = 0
        self._answers: Dict[tuple, Tuple[str, Optional[bytes], int]] = {}

    # ---- counters (b9_depth, b9_depth_bytes, b9_running)
    def depth(self) -> int:
        return len(self.pending)

    def depth_bytes(self) -> int:
        return sum(len(t.payload) for t in self.pending)

    def running(self) -> int:
        # a launch that does not peek claims its window until a fetch commits it or another drain-side call drops it
        return self.window.n if self.window is not None and not self.window.peek else 0

    # ---- answers
    def answer(self, t: Task, handler: str, full_pickle: bool, endpoint: bool) -> Tuple[str, Optional[bytes], int]:
        """(status, result bytes or None, callback kind) of task t in a launch of `handler`, cached per (payload, flags,
        handler, retries, policy): long sequences stay cheap."""
        f = t.flags & ~TF_CANCELLED
        retry = () if endpoint or f & TF_PICKLE else self.retry_for     # the endpoint drain and the function runner have no retry_for
        key = (t.payload, f, handler, full_pickle, endpoint, t.retries, tuple(c.__name__ for c in retry), self.max_retries if retry else 0)
        got = self._answers.get(key)
        if got is None:
            got = self._answers[key] = self._answer(t, f, handler, full_pickle, endpoint, retry)
        return got

    def _answer(self, t, f, handler, full_pickle, endpoint, retry):
        if endpoint:
            # endpoint_accepts (endpoint_device.cuh): HTTP bodies only; run_endpoint_request's outcomes as the drain reports them
            if f != TF_HTTP_BODY:
                return "UNSUPPORTED", None, CB.CB_HOST
            out, body = EP.run_endpoint_request(t.payload, handler)
            status = {EP.OK: "COMPLETE", EP.BAD_REQUEST: "REJECTED", EP.HANDLER_RAISED: "ERROR"}.get(out, "UNSUPPORTED")
            return status, body if out == EP.OK else None, CB.CB_NONE
        if f & TF_PICKLE:
            # B9_DRAIN_PICKLE_FULL answers pickle-framed calls; without it only identity's one-str template is answered,
            # and the generator's pickle calls are never one str
            if not full_pickle:
                return "UNSUPPORTED", None, CB.callback_kind("UNSUPPORTED", None, pickle=True)
            st, res = funcloop.run_function_task(t.payload, handler)
            status = "COMPLETE" if st == funcloop.COMPLETE else "ERROR"
            res = res if status == "COMPLETE" else None
            return status, res, CB.callback_kind(status, res, pickle=True)
        if f & TF_TASK_MSG:
            assert json.loads(t.payload)["task_id"] == str(uuid.UUID(bytes=t.id))
        a = run_retry_loop([t.payload], [t.id], handler, retry_for=retry, max_retries=self.max_retries, retries=[t.retries],
                           http_body=[bool(f & TF_HTTP_BODY)], task_msg=[bool(f & TF_TASK_MSG)])[0]
        return a.status, a.result, CB.callback_kind(a.status, a.result, runner_kwargs(t.payload, f))

    # ---- producer side
    def push_verdict(self, n: int, nbytes: int) -> str:
        """"refuse": the push must fail (B9_ENOSPC); "must": it must succeed; "either": both are allowed.
        The model does not restate where b9_ring_place puts a segment. It must refuse what exceeds the free slots or the
        ring's bytes. It must accept when the bytes the live segments hold (each a b9_seg_span, a segment held whole until
        all its tasks are popped) plus this push's fit in half the ring: the ring then has room for it in one piece
        wherever the segments lie, since the only unused gap, at the ring's end, is shorter than the segment that wrapped."""
        if n > self.ring_tasks - self.depth() or self.depth_bytes() + nbytes > self.ring_bytes:
            return "refuse"
        if sum(s[1] for s in self.segs) + seg_span(nbytes) <= self.ring_bytes // 2:
            return "must"
        return "either"

    def push(self, tasks: Sequence[Task]) -> None:
        self.pending += list(tasks)
        if tasks:
            self.segs.append([len(tasks), seg_span(sum(len(t.payload) for t in tasks))])

    # ---- drain side
    def expire(self, now_ns: int) -> int:
        """b9_expire (expire_kernel, b9gpu.cu; the reference's monitor, dispatch.go:173-230): every pending task with
        0 < expires <= now that is not cancelled yet is cancelled. The sweep covers a claimed window too (DESIGN §4.8)."""
        k = 0
        for t in self.pending:
            if 0 < t.expires <= now_ns and not t.flags & TF_CANCELLED:
                t.flags |= TF_CANCELLED
                k += 1
        return k

    def cancel(self, ids: Sequence[bytes]) -> Tuple[int, List[int]]:
        """b9_cancel (cancel_kernel, cancel.cuh; StopTasks): per requested id the OR over the pending slots holding it of
        CLAIMED (a slot of the claimed window: looked up, never written), ALREADY (cancelled already) or MARKED (cancelled
        now); 0 when no pending slot holds it. Returns (slots marked, outcome per requested id)."""
        want = set(ids)
        word: Dict[bytes, int] = {}
        claimed = min(self.running(), self.depth())
        marked = 0
        for i, t in enumerate(self.pending):
            if t.id not in want:
                continue
            if i < claimed:
                bit = CLAIMED
            elif t.flags & TF_CANCELLED:
                bit = ALREADY
            else:
                t.flags |= TF_CANCELLED
                bit = MARKED
                marked += 1
            word[t.id] = word.get(t.id, 0) | bit
        return marked, [word.get(i, 0) for i in ids]

    def launch(self, handler: str, max_tasks: int, peek: bool = False, full_pickle: bool = False, endpoint: bool = False) -> Window:
        """b9_drain_launch / b9_endpoint_drain_launch: the window is the first min(depth, max_tasks, max_drain_tasks) pending
        tasks, its records those of the tasks not cancelled at the launch, in FIFO order (count mode compacts them). Results
        of an earlier launch that were never fetched are dropped (in an async burst only the last launch is fetched)."""
        n = min(self.depth(), max_tasks, self.max_drain_tasks)
        records, retry = [], []
        for t in self.pending[:n]:
            if t.flags & TF_CANCELLED:
                continue
            status, res, kind = self.answer(t, handler, full_pickle, endpoint)
            # RETRY_LIMIT, RETRY and REJECTED records get no callback: the runner `continue`s before send_callback
            # (runner/taskqueue.py:391-397) and a REJECTED payload never became a task (oracle/pyoracle/callback.py)
            records.append(Record(t.id, status, res, kind))
            if status == "RETRY":
                retry.append(t)
        cb = not endpoint and self.cb_key is not None
        self.window = Window(n, peek, endpoint, records, retry, cb, self.cb_key or b"")
        return self.window

    def fetch(self, callbacks: bool = False, too_small: bool = False, now_s: Tuple[int, int] = (0, 0)) -> Window:
        """b9_drain_fetch(_callbacks). too_small: buffers short of the records (B9_ENOSPC: nothing is consumed, and the
        window stays claimed and fetchable). A fetch that fits commits the window exactly once: a peek changes nothing;
        otherwise its n tasks are popped and the tasks of its RETRY records are pushed again at the tail in record order
        (Dispatcher.RetryTask's RPUSH, dispatch.go:232-285) with retries + 1, the commit's clock as their timestamp and the
        same id, bytes and expiry. Their flags are the ones they were pushed with: a CANCELLED bit that a b9_expire sweep
        set on the claimed window is not carried over (the reference's monitor expires only unclaimed tasks); the kept
        expiry cancels them at the next b9_expire (DESIGN §4.9)."""
        w = self.window
        if w is None:
            raise ModelError(B9_EINVAL, "no drain results are waiting")
        if callbacks and not w.callbacks:
            raise ModelError(B9_EINVAL, "the waiting results come from a launch without a callback pass")
        if too_small:
            raise ModelError(B9_ENOSPC, "the records do not fit")
        self.window = None
        if w.peek:
            return w
        self.pending = self.pending[w.n:]
        self.tasks_drained += w.n
        left = w.n
        while left and self.segs:
            take = min(left, self.segs[0][0])
            self.segs[0][0] -= take
            left -= take
            if self.segs[0][0] == 0:
                self.segs.pop(0)
        again = [Task(t.id, t.payload, t.flags & ~TF_CANCELLED, t.retries + 1, t.expires, now_s, True) for t in w.retry]
        if again:
            self.pending += again
            # (one segment, or two split at a task boundary around the ring's end: one more alignment pad at most)
            self.segs.append([len(again), seg_span(sum(len(t.payload) for t in again)) + SEG_ALIGN])
        return w

    def wire_window(self, max_tasks: int) -> List[Task]:
        """b9_wire_encode(_full): records of the first pending tasks, which stay pending; an outstanding launch is dropped."""
        self.window = None
        return list(self.pending[:min(self.depth(), max_tasks, self.max_drain_tasks)])

    def set_retry_policy(self, classes: Sequence[type], max_retries: int) -> None:
        self.retry_for = tuple(classes)
        self.max_retries = max_retries

    def set_callback_policy(self, key: Optional[bytes]) -> None:
        self.cb_key = key

    def snapshot(self) -> tuple:
        """Everything the model holds, comparable across replays."""
        w = self.window
        return (tuple((t.id, t.payload, t.flags, t.retries, t.expires, t.ts, t.repushed) for t in self.pending),
                tuple(tuple(s) for s in self.segs), self.tasks_drained, self.retry_for, self.max_retries, self.cb_key,
                None if w is None else (w.n, w.peek, w.endpoint, tuple((r.id, r.status, r.result, r.kind) for r in w.records)))


def runner_kwargs(payload: bytes, flags: int) -> Optional[dict]:
    """The kwargs the runner would call the handler with (None when the payload never becomes a task)."""
    try:
        if flags & TF_TASK_MSG:
            return json.loads(payload)["kwargs"]
        if flags & TF_HTTP_BODY:
            return serialize_http_payload(payload)[1]
        return go_unmarshal_task_payload(payload)[1]
    except (GoJSONError, InvalidRequestPayload, ValueError, KeyError):
        return None


def expected_digest(rec: Record, key: bytes, ts: int) -> bytes:
    """SignPayload (pkg/auth/sign.go:17-35) over the runner's body for a B9_CB_POST record under a key, else 32 zero bytes."""
    if rec.kind != CB.CB_POST or not key:
        return bytes(32)
    return hmac.new(key, CB.sign_message(CB.callback_body(rec.result), ts), hashlib.sha256).digest()


# ---------------------------------------------------------------------------------------------------- the corpus
def task_id(salt: int, k: int) -> bytes:
    return uuid.UUID(int=(salt << 64) | k).bytes


@dataclass
class Item:
    payload: bytes
    flags: int
    id: Optional[bytes] = None              # a TaskMessage record names its own id


def corpus() -> List[Item]:
    """Payloads of every framing the queue takes: SDK strings with escapes and non-ASCII, json_sum documents with floats,
    the retry-raising calls of tests/test_gpu_retry.py, HTTP bodies, TaskMessage records, pickle blobs and callback_url
    keyword arguments."""
    from tests.test_retry_on_host import CLASS_ARGS
    items: List[Item] = []
    strings = ["plain", 'q"uote \\ back\nline\ttab', "héllo wörld €", "\U0001f600 emoji", "<a>&amp;</a>", "", "x" * 200,
               " sep ", "ctl \x01\x1f"]
    items += [Item(sdk_put_payload(s), 0) for s in strings]
    docs = [{"values": [0.5, 1.25, -2.75]}, {"values": [1e300, 1e300]}, {"values": [0.1] * 7}, {"values": [3, 4.5e-3, 1e10]},
            {"values": [1, 2, 3]}, {"values": [-1e308, -1e308]}, {"values": []}, {"values": [2.5e-300, 7]}]
    items += [Item(sdk_put_payload(d), 0) for d in docs]
    calls = [a for h in HANDLERS for a in CLASS_ARGS[h] if "\ud83d" not in json.dumps(a)]
    items += [Item(sdk_put_payload(*a), 0) for a in calls]
    items += [Item(sdk_put_payload(*a, extra=1), 0) for a in calls[::3]]
    bodies = [json.dumps({"args": a}).encode() for a in calls[::2]] + [json.dumps({"args": ["café"], "kwargs": {}}).encode(),
                                                                     b'{"values": [1, 2.5]}', b"{}", b"not json", b"[1]"]
    items += [Item(b, TF_HTTP_BODY) for b in bodies]
    items += [Item(b"not json", 0), Item(b'{"args": ["unterminated"', 0)]
    items += [Item(sdk_put_payload("x", callback_url="http://o.invalid/cb"), 0), Item(sdk_put_payload({"values": [1]}, callback_url="u"), 0),
              Item(sdk_put_payload("x", callback_url=""), 0)]
    rec_calls = [("rec",), ({"values": [4, 0.5]},), ("réc \"q\"",), ({"k": 1},), (None,)]
    rec_ids = [task_id(0xC0DE, k) for k in range(len(rec_calls))]
    for rid, w in zip(rec_ids, run_task_loop([sdk_put_payload(*a) for a in rec_calls], rec_ids, "identity", keep_wire=True)):
        items.append(Item(w.wire, TF_TASK_MSG, rid))
    # pickle calls that are never one str (identity answers those without B9_DRAIN_PICKLE_FULL) and that no handler declines
    from tests.pickle_corpus import declined, frame_one
    for v in [5, [1, 2], {"values": [1, 2.5]}, {"a": 1}, None, 2.5, {"values": "ab"}, [b"x"]]:
        blob = frame_one(v)
        if not any(declined(blob, h) for h in HANDLERS):
            items.append(Item(blob, TF_PICKLE))
    return items


# ---------------------------------------------------------------------------------------------------- operations
# op kinds, each a dict with "op" and its arguments; a push records whether the device took it ("accepted")
PUSH_KINDS = ("push_batch", "push_scattered", "submit")


class OpGen:
    """Draws weighted operations from the model's state: the same seed, shape and device outcomes give the same log."""

    def __init__(self, seed: int, items: List[Item], model: QueueModel, tiny: bool):
        self.rng = random.Random(seed)
        self.seed = seed
        self.items = items
        self.model = model
        self.tiny = tiny
        self.k = 0                           # ids drawn so far
        self.now = 1_000_000
        self.gone: List[bytes] = []          # ids that left the queue
        self.bursting = 0                    # async launches still to come in the current burst

    def _tasks(self, n: int, kind: str) -> List[dict]:
        out = []
        for _ in range(n):
            it = self.rng.choice(self.items)
            self.k += 1
            tid = it.id if it.id is not None else task_id(self.seed + 1, self.k)
            flags = it.flags if kind != "push_scattered" else 0      # (b9_batch_push_v takes no flags)
            if kind == "push_batch":
                flags |= TF_CANCELLED if self.rng.random() < 0.08 else 0
                retries = self.rng.choice([0, 0, 0, 1, 2, 3])
                r = self.rng.random()
                expires = 0 if r < 0.5 else max(1, self.now + self.rng.randint(-3000, 12000))
            else:
                retries, expires = 0, 0
                if kind == "submit":
                    flags |= TF_CANCELLED if self.rng.random() < 0.08 else 0
            out.append(dict(id=tid.hex(), item=self.items.index(it), flags=flags, retries=retries, expires=expires))
        return out

    def next(self) -> dict:
        rng, m = self.rng, self.model
        self.now += 1000
        w = m.window
        if self.k == 0 and rng.random() < 0.75:          # most runs start under a retry policy
            self.k = 1
            return dict(op="retry_policy", classes=sorted(rng.sample(range(len(RETRY_CLASSES)), 3)), max_retries=rng.randint(1, 4))
        if self.bursting:
            self.bursting -= 1
            return self._launch(wait=False)
        choices = [("push", 22), ("cancel", 9), ("expire", 8), ("launch", 20), ("retry_policy", 3), ("cb_policy", 3), ("wire", 2)]
        if w is not None:
            choices += [("fetch", 45)]
        op = rng.choices([c for c, _ in choices], [wt for _, wt in choices])[0]
        if op == "push":
            kind = rng.choices(PUSH_KINDS, [6, 2, 2])[0]
            n = rng.randint(1, 6 if self.tiny else 120) if kind != "submit" else rng.randint(1, 4)
            if self.tiny and kind != "submit" and rng.random() < 0.35:
                n = max(1, m.ring_tasks - m.depth())      # fill the slots: the tiny ring is often exactly full
            tasks = self._tasks(n, kind)
            if kind == "submit":          # b9_submit's arena holds half the ring: a submit is only tried where it must fit
                nb = sum(len(self.items[t["item"]].payload) for t in tasks)
                if m.push_verdict(n, nb) != "must" or nb > m.ring_bytes // 4:
                    kind = "push_batch"
            return dict(op=kind, tasks=tasks, ts=1_700_000_000 + self.now // 1000)
        if op == "cancel":
            pool = [("pending", [t.id for t in m.pending]), ("claimed", [t.id for t in m.pending[:m.running()]]),
                    ("repushed", [t.id for t in m.pending if t.repushed]), ("gone", self.gone[-50:])]
            ids = []
            for _ in range(rng.randint(1, 8)):
                name, ids_of = rng.choice(pool)
                if ids_of:
                    ids.append(rng.choice(ids_of))
                else:
                    ids.append(task_id(0xDEAD, rng.randrange(1 << 30)))
            if ids and rng.random() < 0.3:
                ids.append(rng.choice(ids))                  # a duplicate in one call
            return dict(op="cancel", ids=[i.hex() for i in ids])
        if op == "expire":
            return dict(op="expire", now=self.now + rng.randint(-2000, 6000))
        if op == "launch":
            r = rng.random()
            if r < 0.25:
                self.bursting = rng.randint(1, 4)          # a burst of 2-5 async launches
                return self._launch(wait=False)
            return self._launch(wait=True, peek=r > 0.8)
        if op == "retry_policy":
            if rng.random() < 0.25:
                return dict(op="retry_policy", classes=[], max_retries=0)
            cls = rng.sample(range(len(RETRY_CLASSES)), rng.randint(1, 3))
            return dict(op="retry_policy", classes=sorted(cls), max_retries=rng.randint(0, 4))
        if op == "cb_policy":
            return dict(op="cb_policy", key=rng.choice([None, "", "6b6579", (b"workspace-key-%d" % rng.randrange(9)).hex()]))
        if op == "wire":
            return dict(op="wire", max_tasks=rng.randint(1, 64))
        # fetch: a too-small one first, sometimes; callbacks when the launch ran the pass (and rarely when it did not)
        cbk = w.callbacks if rng.random() < 0.95 else not w.callbacks
        sizes = [len(r.result or b"") for r in w.records]
        small = None
        if rng.random() < 0.5:
            if len(w.records) >= 2 and rng.random() < 0.5:
                small = ["tasks", len(w.records) - 1]
            elif sum(sizes) >= 2:
                small = ["bytes", sum(sizes) - 1]
        return dict(op="fetch", callbacks=cbk, small=small)

    def _launch(self, wait: bool, peek: bool = False) -> dict:
        rng = self.rng
        handler = rng.choice(HANDLERS)
        r = rng.random()
        endpoint = r < 0.12
        full = (not endpoint) and r > 0.7
        limit = self.model.max_drain_tasks
        max_tasks = rng.choice([1, 2, 3, rng.randint(1, limit), limit, 1 << 22])
        return dict(op="launch", handler=handler, max_tasks=max_tasks, peek=peek or (not wait and rng.random() < 0.2),
                    wait=wait, full_pickle=full, endpoint=endpoint)


def make_tasks(op: dict, items: List[Item]) -> List[Task]:
    ts = op.get("ts", 0) if op["op"] == "push_batch" else 0
    return [Task(bytes.fromhex(t["id"]), items[t["item"]].payload, t["flags"], t["retries"], t["expires"], (ts, ts)) for t in op["tasks"]]


def apply(model: QueueModel, op: dict, items: List[Item]):
    """Plays one logged operation on the model; -> the model's answer (see QueueModel), or a ModelError it raises."""
    kind = op["op"]
    if kind in PUSH_KINDS:
        tasks = make_tasks(op, items)
        if op.get("accepted", model.push_verdict(len(tasks), sum(len(t.payload) for t in tasks)) != "refuse"):
            model.push(tasks)
            return True
        return False
    if kind == "cancel":
        return model.cancel([bytes.fromhex(i) for i in op["ids"]])
    if kind == "expire":
        return model.expire(op["now"])
    if kind == "launch":
        return model.launch(op["handler"], op["max_tasks"], op["peek"], op["full_pickle"], op["endpoint"])
    if kind == "fetch":
        if op["small"] is not None:           # buffers one record or one byte short first: B9_ENOSPC, then the fetch that fits
            try:
                model.fetch(op["callbacks"], too_small=True)
            except ModelError as e:
                if e.code != B9_ENOSPC:
                    raise
        return model.fetch(op["callbacks"], False, tuple(op.get("t", (0, 0))))
    if kind == "retry_policy":
        model.set_retry_policy([RETRY_CLASSES[c] for c in op["classes"]], op["max_retries"])
        return None
    if kind == "cb_policy":
        model.set_callback_policy(None if op["key"] is None else bytes.fromhex(op["key"]))
        return None
    if kind == "wire":
        return model.wire_window(op["max_tasks"])
    raise ValueError(kind)


def run_model(seed: int, n_ops: int, ring_bytes: int, ring_tasks: int, tiny: bool, items: Optional[List[Item]] = None):
    """The CPU-only run of a seed: -> (model, log). A push's outcome follows push_verdict ("either" takes the push)."""
    items = items if items is not None else corpus()
    m = QueueModel(ring_bytes, ring_tasks, ring_tasks)
    gen = OpGen(seed, items, m, tiny)
    log = []
    for _ in range(n_ops):
        op = gen.next()
        try:
            before = [t.id for t in m.pending]
            apply(m, op, items)
            now = set(t.id for t in m.pending)
            gen.gone += [i for i in before if i not in now]
        except ModelError:
            pass
        log.append(op)
    return m, log
