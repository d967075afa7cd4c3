"""GPU: the queue's calls interleaved against tests/queue_model.py. Random sequences of pushes, submits, cancels,
expiries, blocking / peek / async-burst launches of every handler (with B9_DRAIN_PICKLE_FULL and the endpoint drain
sometimes), fetches refused with B9_ENOSPC first, retry and callback policies changed between launches and wire
records of the pending window, on a tiny ring that wraps every few calls and a mid-sized one. After every call the
fetched records (id, status, bytes, callback kind and digest), depth, running, depth_bytes and the tasks_drained /
bytes_d2h deltas must be the model's. A failure names the seed, the step and the operation log, which replays."""
import json
import time
import uuid
from collections import Counter

import numpy as np
import pytest

from beta9_b200 import _lib as L
from beta9_b200.device_queue import STATUS_NAMES, DeviceQueue
from oracle.pyoracle.gojson import GoJSONError, go_unmarshal_task_payload
from oracle.pyoracle.httpserialize import InvalidRequestPayload, serialize_http_payload
from tests import queue_model as QM

pytestmark = pytest.mark.gpu
KEY = b"workspace-signing-key-0123456789"


@pytest.fixture(scope="module")
def items():
    return QM.corpus()


def as_ids(ids):
    return np.frombuffer(b"".join(ids), np.uint8).reshape(-1, 16)


class Driver:
    """One DeviceQueue and its model, driven by the same operations; counts the interactions the random runs reach."""

    def __init__(self, items, ring_bytes, ring_tasks, max_result_bytes=1 << 22):
        self.items = items
        self.q = DeviceQueue(ring_bytes=ring_bytes, ring_tasks=ring_tasks, max_drain_tasks=ring_tasks, max_result_bytes=max_result_bytes)
        self.m = QM.QueueModel(ring_bytes, ring_tasks, ring_tasks)
        self.launch_t = (0, 0)
        self.seen = Counter()
        self.gone = []

    def close(self):
        self.q.close()

    # ---- one operation on both sides
    def do(self, op):
        q, m = self.q, self.m
        kind = op["op"]
        s0 = q.stats()
        drained0 = m.tasks_drained
        d2h = 0
        res = None
        before = [t.id for t in m.pending]
        if kind in QM.PUSH_KINDS:
            tasks = QM.make_tasks(op, self.items)
            verdict = m.push_verdict(len(tasks), sum(len(t.payload) for t in tasks))
            try:
                self._push(kind, op, tasks)
                op["accepted"] = True
            except L.B9Error as e:
                assert e.code == L.B9_ENOSPC, e
                op["accepted"] = False
            assert verdict != {True: "refuse", False: "must"}[op["accepted"]], (verdict, op["accepted"])
            self.seen["push refused"] += not op["accepted"]
            QM.apply(m, op, self.items)
        elif kind == "cancel":
            ids = [bytes.fromhex(i) for i in op["ids"]]
            claimed = {t.id for t in m.pending[:m.running()]}
            marked, out = q.cancel(as_ids(ids))
            want = QM.apply(m, op, self.items)
            assert (marked, out.tolist()) == (want[0], list(want[1]))
            res = want
            self.seen["cancel of a claimed id"] += any(i in claimed for i in ids)
        elif kind == "expire":
            win = [t for t in m.pending[:m.running()] if not t.flags & QM.TF_CANCELLED]
            got = q.expire(op["now"])
            assert got == QM.apply(m, op, self.items)
            self.seen["expire inside a claimed window"] += any(t.flags & QM.TF_CANCELLED for t in win)
        elif kind == "launch":
            t0 = int(time.time())
            got = q.drain_launch(op["handler"], op["max_tasks"], peek=op["peek"], wait=op["wait"], full_pickle=op["full_pickle"],
                                 endpoint=op["endpoint"])
            self.launch_t = (t0, int(time.time()) + 1)
            w = QM.apply(m, op, self.items)
            assert got == (len(w.records) if op["wait"] else w.n)
            self.seen["async launch"] += not op["wait"]
        elif kind == "fetch":
            d2h = self._fetch(op)
        elif kind == "retry_policy":
            q.set_retry_policy([QM.RETRY_CLASSES[c] for c in op["classes"]], op["max_retries"])
            QM.apply(m, op, self.items)
        elif kind == "cb_policy":
            q.set_callback_policy(None if op["key"] is None else bytes.fromhex(op["key"]))
            QM.apply(m, op, self.items)
        elif kind == "wire":
            r = q.wire_encode("ws", "stub-1", max_tasks=op["max_tasks"], full=True)
            self._check_wire(r, QM.apply(m, op, self.items))
            d2h = r.payload.size + r.n * QM.RECORD_BYTES
        now = {t.id for t in m.pending}
        self.gone += [i for i in before if i not in now]
        s1 = q.stats()
        assert (q.depth(), q.depth_bytes(), q.running()) == (m.depth(), m.depth_bytes(), m.running())
        assert s1.tasks_drained - s0.tasks_drained == m.tasks_drained - drained0
        assert s1.bytes_d2h - s0.bytes_d2h == d2h
        return res

    def _push(self, kind, op, tasks):
        q = self.q
        ids = as_ids([t.id for t in tasks])
        if kind == "push_batch":
            off = np.zeros(len(tasks) + 1, np.uint64)
            np.cumsum([len(t.payload) for t in tasks], out=off[1:])
            q.push_batch(ids, np.frombuffer(b"".join(t.payload for t in tasks), np.uint8), off,
                         timestamp_unix=np.full(len(tasks), op["ts"], np.int64), expires_unix_ns=np.array([t.expires for t in tasks], np.int64),
                         retries=np.array([t.retries for t in tasks], np.uint8), flags=np.array([t.flags for t in tasks], np.uint8))
        elif kind == "push_scattered":
            bufs = [np.frombuffer(t.payload or b"\0", np.uint8).copy() for t in tasks]
            q.push_scattered(ids, np.array([b.ctypes.data for b in bufs], np.uint64), np.array([len(t.payload) for t in tasks], np.uint32))
            q.sync()
        else:
            for t in tasks:
                q.submit(t.id, t.payload, t.flags)
            assert q.flush() == len(tasks) and q.buffered() == 0

    def _fetch(self, op):
        q, m = self.q, self.m
        w = m.window
        if op["small"] is not None:
            what, k = op["small"]
            s0 = q.stats()
            with pytest.raises(L.B9Error) as e:
                q.fetch(callbacks=op["callbacks"], **({"cap_tasks": k} if what == "tasks" else {"cap_bytes": k}))
            want = L.B9_EINVAL if w is None or (op["callbacks"] and not w.callbacks) else L.B9_ENOSPC
            assert e.value.code == want
            if want == L.B9_ENOSPC:
                assert (q.depth(), q.running(), q.stats().bytes_d2h, q.stats().tasks_drained) == (m.depth(), m.running(), s0.bytes_d2h, s0.tasks_drained)
        full_ring = m.depth() == m.ring_tasks
        t0 = int(time.time())
        try:
            r = q.fetch(callbacks=op["callbacks"])
        except L.B9Error as e:
            op["t"] = (t0, int(time.time()) + 1)
            with pytest.raises(QM.ModelError) as me:
                QM.apply(m, op, self.items)
            assert e.code == me.value.code
            return 0
        op["t"] = (t0, int(time.time()) + 1)
        w = QM.apply(m, op, self.items)
        assert r.n == len(w.records) and r.n_popped == w.n
        got = [(bytes(r.task_ids[i]), STATUS_NAMES[int(r.status[i])], r.result(i)) for i in range(r.n)]
        assert got == [(x.id, x.status, x.result) for x in w.records]
        cb_bytes = 0
        if op["callbacks"]:
            keyed = bool(w.key)
            ts = int(r.cb_timestamp)
            assert (self.launch_t[0] <= ts <= self.launch_t[1]) if keyed else ts == 0
            assert r.cb_kind.tolist() == [x.kind for x in w.records]
            for i, x in enumerate(w.records):
                assert r.cb_digest[i].tobytes() == QM.expected_digest(x, w.key, ts), i
            cb_bytes = r.n * (1 + (32 if keyed else 0))
            self.seen["count mode with callbacks"] += w.n > r.n
        if w.retry and not w.peek:
            self.seen["re-push"] += 1
            self.seen["B9_ENOSPC fetch then re-push"] += op["small"] is not None
            self.seen["re-push into an exactly full ring"] += full_ring
        return r.payload.size + r.n * QM.RECORD_BYTES + cb_bytes

    def _check_wire(self, r, tasks):
        """b9_wire_encode_full of the pending window: one record per task in FIFO order; an encoded record carries the slot's
        retries and timestamp (a re-pushed task: retries + 1 and the commit's clock)."""
        assert r.n == len(tasks) and [bytes(i) for i in r.task_ids] == [t.id for t in tasks]
        for i, t in enumerate(tasks):
            st = int(r.status[i])
            if t.flags & (QM.TF_TASK_MSG | QM.TF_PICKLE):
                assert st == L.ST_UNSUPPORTED
                continue
            try:
                (serialize_http_payload if t.flags & QM.TF_HTTP_BODY else go_unmarshal_task_payload)(t.payload)
            except (GoJSONError, InvalidRequestPayload):
                assert st == L.ST_REJECTED
                continue
            assert st in (L.ST_COMPLETE, L.ST_UNSUPPORTED), st
            if st == L.ST_COMPLETE:
                rec = json.loads(r.result(i))
                assert rec["task_id"] == str(uuid.UUID(bytes=t.id)) and rec["retries"] == t.retries
                assert t.ts[0] <= rec["timestamp"] <= t.ts[1], (rec["timestamp"], t.ts)
                self.seen["wire record of a re-pushed task"] += t.repushed


def run_seed(items, seed, n_ops, ring_bytes, ring_tasks, tiny):
    d = Driver(items, ring_bytes, ring_tasks)
    gen = QM.OpGen(seed, items, d.m, tiny)
    log = []
    try:
        for step in range(n_ops):
            op = gen.next()
            log.append(op)
            try:
                d.do(op)
            except QM.ModelError as e:                   # a call the model refuses must be refused by the library too
                raise AssertionError(f"the library took a call the model refuses: {e}")
            gen.gone = d.gone
            d.seen[op["op"]] += 1
    except Exception as e:
        raise AssertionError(f"seed {seed} ({ring_bytes} B, {ring_tasks} slots), step {len(log) - 1}: {e!r}\n"
                             f"op log: {json.dumps(log)}") from e
    finally:
        d.close()
    return d.seen


SEEDS = [(s, 1 << 12, (16, 32, 64)[s % 3], True) for s in range(12)] + [(s, 1 << 20, 1 << 12, False) for s in range(100, 112)]


def test_random_sequences_against_the_model(items):
    """24 seeds of 300 operations: 12 on a 4 KiB ring of 16 / 32 / 64 slots, 12 on a 1 MiB ring of 4 Ki slots."""
    total = Counter()
    for seed, rb, rt, tiny in SEEDS:
        seen = run_seed(items, seed, 300, rb, rt, tiny)
        total += seen
    print("\nqueue model: seeds %s, 300 operations each; %s" % ([s for s, *_ in SEEDS], json.dumps(dict(sorted(total.items())))))
    for k in ("B9_ENOSPC fetch then re-push", "expire inside a claimed window", "re-push into an exactly full ring",
              "count mode with callbacks", "cancel of a claimed id", "wire record of a re-pushed task"):
        assert total[k] >= 10, (k, total[k])


# ---------------------------------------------------------------------------------------------------- named interactions
def sdk(*a, **kw):
    return QM.sdk_put_payload(*a, **kw)


KEYERR = sdk({"v": 1})                      # json_sum raises KeyError
OK = sdk({"values": [1, 2.5]})


def driver(items, ring_bytes=1 << 16, ring_tasks=64):
    return Driver(items, ring_bytes, ring_tasks)


def push(d, payloads, salt, **kw):
    op = dict(op="push_batch", ts=1_700_000_000, tasks=[])
    for k, p in enumerate(payloads):
        it = len(d.items)
        d.items.append(QM.Item(p, 0))
        op["tasks"].append(dict(id=QM.task_id(salt, k).hex(), item=it, flags=kw.get("flags", 0), retries=kw.get("retries", 0),
                                expires=kw.get("expires", 0)))
    d.do(op)
    assert op["accepted"]
    return [QM.task_id(salt, k) for k in range(len(payloads))]


def launch(d, handler="json_sum", max_tasks=64, **kw):
    op = dict(op="launch", handler=handler, max_tasks=max_tasks, peek=kw.get("peek", False), wait=kw.get("wait", True),
              full_pickle=False, endpoint=False)
    d.do(op)


def fetch(d, small=None, callbacks=False):
    op = dict(op="fetch", callbacks=callbacks, small=small)
    d.do(op)
    return op


def test_retry_with_expire_between_launch_and_fetch(items):
    """An expire sweep of the claimed window cancels nothing that is re-pushed: the retried task is pending, uncancelled,
    with retries + 1 and its expiry, drains RETRY again, and the next expire cancels it."""
    d = driver(list(items))
    try:
        d.do(dict(op="retry_policy", classes=[QM.RETRY_CLASSES.index(KeyError)], max_retries=3))
        push(d, [KEYERR, OK], 1, expires=500)
        launch(d)
        d.do(dict(op="expire", now=600))
        assert d.m.pending[0].flags & QM.TF_CANCELLED
        fetch(d)
        assert d.q.depth() == 1 and d.m.pending[0].flags == 0 and d.m.pending[0].retries == 1
        launch(d, peek=True)
        assert [x.status for x in d.m.window.records] == ["RETRY"]
        fetch(d)
        d.do(dict(op="expire", now=600))
        launch(d)
        assert d.m.window.records == []
        fetch(d)
        assert d.q.depth() == 0
    finally:
        d.close()


def test_retry_with_enospc_fetch_then_larger_fetch(items):
    d = driver(list(items))
    try:
        d.do(dict(op="retry_policy", classes=[QM.RETRY_CLASSES.index(KeyError)], max_retries=2))
        push(d, [KEYERR, OK, KEYERR, OK, KEYERR], 2)
        launch(d)
        fetch(d, small=["tasks", 4])                       # one record short, then the fetch that fits: one re-push
        assert d.q.depth() == 3 and [t.retries for t in d.m.pending] == [1, 1, 1]
        fetch_twice = dict(op="fetch", callbacks=False, small=None)
        d.do(fetch_twice)                                  # nothing waits any more: B9_EINVAL, nothing re-pushed again
        assert d.q.depth() == 3
        launch(d)
        fetch(d, small=["tasks", 2])
        assert d.q.depth() == 3 and [t.retries for t in d.m.pending] == [2, 2, 2]
        d.do(dict(op="wire", max_tasks=8))
    finally:
        d.close()


def test_retry_with_an_async_burst(items):
    d = driver(list(items))
    try:
        d.do(dict(op="retry_policy", classes=[QM.RETRY_CLASSES.index(KeyError)], max_retries=3))
        push(d, [KEYERR] * 6 + [OK] * 2, 3)
        for mt in (6, 2, 4):
            launch(d, max_tasks=mt, wait=False)
        fetch(d)                                           # only the last launch (4 tasks) is fetched and re-pushed
        assert d.q.depth() == 8 and [t.retries for t in d.m.pending] == [0, 0, 0, 0, 1, 1, 1, 1]
    finally:
        d.close()


def test_retry_with_cancel_of_a_claimed_id_then_of_its_copy(items):
    d = driver(list(items))
    try:
        d.do(dict(op="retry_policy", classes=[QM.RETRY_CLASSES.index(KeyError)], max_retries=3))
        ids = push(d, [KEYERR, OK], 4)
        launch(d, wait=False)
        assert d.do(dict(op="cancel", ids=[ids[0].hex(), ids[1].hex()])) == (0, [QM.CLAIMED, QM.CLAIMED])
        fetch(d)                                           # the claimed task comes back RETRY and is pushed again
        assert d.q.depth() == 1
        assert d.do(dict(op="cancel", ids=[ids[0].hex()])) == (1, [QM.MARKED])
        launch(d)
        fetch(d)
        assert d.q.depth() == 0
    finally:
        d.close()


@pytest.mark.parametrize("key", [KEY, b""])
def test_callback_policy_with_retries_counts_the_callback_read_back(items, key):
    """bytes_d2h of a fetch that re-pushes counts the kinds (and the digests under a key), like a fetch that does not."""
    d = driver(list(items))
    try:
        d.do(dict(op="retry_policy", classes=[QM.RETRY_CLASSES.index(KeyError)], max_retries=3))
        d.do(dict(op="cb_policy", key=key.hex()))
        push(d, [KEYERR, OK, KEYERR, sdk({"values": [1e308, 1e308]})], 5)
        s0 = d.q.stats()
        launch(d)
        fetch(d, callbacks=True)                           # Driver.do checks the delta: records + 4 x (1 + 32 if keyed)
        assert d.q.stats().bytes_d2h - s0.bytes_d2h >= 4 * (QM.RECORD_BYTES + 1 + (32 if key else 0))
        assert d.q.depth() == 2
    finally:
        d.close()


@pytest.mark.parametrize("handler,n", [("identity", 3000), ("vadd_f32", 3000), ("json_sum", 1000), ("json_sum", 260_000)])
def test_count_mode_callbacks_on_a_wrapped_ring(items, handler, n):
    """Cancelled slots in the window (records compacted) under a keyed callback policy, after the slot ring has wrapped;
    json_sum at 1000 tasks runs 4-task tiles and at 260 k tasks 8-task tiles."""
    pool = [sdk("s%d" % k) for k in range(7)] + [sdk("é\"\\"), sdk("AACAPwAAAEAAAIA/AAAAQA=="), sdk("AAA*"), sdk({"values": [3, 0.5]}),
                                                  sdk({"v": 1}), sdk(1, 2), b"not json"]
    slots = 1 << 19 if n > 100_000 else 1 << 13
    d = Driver(list(items), 1 << 25, slots, max_result_bytes=1 << 26)
    try:
        base = len(d.items)
        d.items += [QM.Item(p, 0) for p in pool]
        rng = np.random.default_rng(n)

        def batch(m, salt):
            op = dict(op="push_batch", ts=1_700_000_000, tasks=[])
            for k in range(m):
                op["tasks"].append(dict(id=QM.task_id(salt, k).hex(), item=base + int(rng.integers(len(pool))),
                                        flags=QM.TF_CANCELLED if rng.random() < 0.1 else 0, retries=0, expires=0))
            d.do(op)
            assert op["accepted"]
        batch(slots - n // 2, 60)                    # advance the head so that the next window wraps the slot ring
        launch(d, handler, 1 << 22)
        fetch(d)
        d.do(dict(op="cb_policy", key=KEY.hex()))
        batch(n, 61)
        d.do(dict(op="cancel", ids=[QM.task_id(61, k).hex() for k in range(0, n, 13)]))
        launch(d, handler, 1 << 22)
        w = d.m.window
        assert w.n == n and len(w.records) < n
        fetch(d, callbacks=True)
        assert d.q.depth() == 0
    finally:
        d.close()
