"""GPU tests of the retry policy (b9_set_retry_policy): a task whose handler raised a `retry_for` class comes back RETRY
and is pushed again on the device at the fetch (retries + 1, RPUSH at the tail), or RETRY_LIMIT once its retries are
used up (runner/taskqueue.py:352-393, Dispatcher.RetryTask in pkg/task/dispatch.go:232-285). Every sequence of answers
over the drains that empty a queue must equal tests/retry_oracle.py's single runner."""
import binascii
import json
import threading
import time
import uuid

import numpy as np
import pytest

from beta9_b200 import _lib as L
from beta9_b200.device_queue import EXC_BITS, STATUS_NAMES, DeviceQueue
from oracle.pyoracle import loop
from oracle.pyoracle.loop import sdk_put_payload
from tests.retry_oracle import run_retry_loop
from tests.test_retry_on_host import CLASS_ARGS

pytestmark = pytest.mark.gpu
HANDLERS = ["identity", "crc32", "vadd_f32", "json_sum"]
VALID = {"identity": [["hello"], [3], [{"a": [1, 2]}]], "crc32": [["hello"], ["é€"]],
         "vadd_f32": [["AAAAAAAAAAA="], ["AACAPwAAAEAAAIA/AAAAQA=="]], "json_sum": [[{"values": [1, 2, 3]}], [{"values": [0.5, 1]}]]}


def small_queue(ring_bytes=1 << 22, ring_tasks=1 << 12):
    return DeviceQueue(ring_bytes=ring_bytes, ring_tasks=ring_tasks, max_drain_tasks=ring_tasks, max_result_bytes=1 << 22)


def ids_for(n, salt):
    return np.frombuffer(b"".join(uuid.UUID(int=(salt << 64) | i).bytes for i in range(n)), np.uint8).reshape(n, 16)


def build_corpus(handler, salt):
    """Errors of every class a handler raises mixed with valid tasks, in the three framings: SDK payloads, HTTP bodies
    (B9_TF_HTTP_BODY) and the TaskMessage records Go writes (B9_TF_TASK_MSG). -> payloads, ids [n,16], flags, retries"""
    calls = [a for a in CLASS_ARGS[handler] if "\ud83d" not in json.dumps(a)] + VALID[handler]
    payloads, flags = [], []
    for a in calls:
        payloads.append(sdk_put_payload(*a)); flags.append(0)
        payloads.append(sdk_put_payload(*a, extra=1)); flags.append(0)
        payloads.append(json.dumps({"args": a}).encode()); flags.append(L.TF_HTTP_BODY)
    ids = ids_for(len(payloads) + len(calls), salt)
    live = loop.run_task_loop([sdk_put_payload(*a) for a in calls], [bytes(ids[len(payloads) + i]) for i in range(len(calls))],
                              "identity", keep_wire=True)
    for w in live:
        payloads.append(w.wire); flags.append(L.TF_TASK_MSG)
    rng = np.random.default_rng(salt)
    order = rng.permutation(len(payloads))
    payloads = [payloads[i] for i in order]
    ids = ids[order]
    flags = np.array([flags[i] for i in order], np.uint8)
    retries = rng.integers(0, 3, len(payloads)).astype(np.uint8) * (rng.random(len(payloads)) < 0.3)
    return payloads, ids, flags, retries


def push(q, payloads, ids, flags=None, retries=None):
    off = np.zeros(len(payloads) + 1, np.uint64)
    np.cumsum([len(p) for p in payloads], out=off[1:])
    q.push_batch(ids, np.frombuffer(b"".join(payloads), np.uint8), off, flags=flags, retries=retries)


def drain_all(q, handler, window, check=None):
    """Drains until the queue is empty; -> [(id, status, result)]. Checks depth / running after every fetch."""
    out = []
    for _ in range(10_000):
        d0 = q.depth()
        if d0 == 0:
            return out
        r = q.drain(handler, window)
        recs = r.records()
        n_retry = sum(1 for _, s, _ in recs if s == "RETRY")
        assert q.depth() == d0 - r.n_popped + n_retry and q.running() == 0
        for _, s, res in recs:
            assert s != "UNSUPPORTED"
            if s in ("RETRY", "RETRY_LIMIT"):
                assert res is None
        out += recs
    raise AssertionError("the queue did not empty")


def oracle_answers(payloads, ids, flags, retries, handler, classes, max_retries):
    want = run_retry_loop(payloads, [bytes(i) for i in ids], handler, retry_for=classes, max_retries=max_retries,
                          retries=[int(r) for r in retries], http_body=[bool(f & L.TF_HTTP_BODY) for f in flags],
                          task_msg=[bool(f & L.TF_TASK_MSG) for f in flags])
    return [(a.task_id, a.status, a.result) for a in want]


MASKS = [[c] for c in EXC_BITS] + [list(EXC_BITS), []]


@pytest.mark.parametrize("handler", HANDLERS)
def test_every_mask_and_limit_equals_the_oracle_loop(handler):
    q = small_queue()
    payloads, ids, flags, retries = build_corpus(handler, 1 + HANDLERS.index(handler))
    try:
        for classes in MASKS:
            for max_retries in (0, 1, 3):
                q.set_retry_policy(classes, max_retries)
                push(q, payloads, ids, flags, retries)
                got = drain_all(q, handler, window=7)
                want = oracle_answers(payloads, ids, flags, retries, handler, classes, max_retries)
                assert got == want, (classes, max_retries)
    finally:
        q.close()


def test_repushed_tasks_keep_bytes_and_show_retries_and_timestamp():
    q = small_queue()
    try:
        calls = [[{}], [{"values": [1]}], [{"v": 2}], [{"values": [2]}]]
        payloads = [sdk_put_payload(*a) for a in calls]
        ids = ids_for(len(payloads), 77)
        q.set_retry_policy([KeyError], 3)
        push(q, payloads, ids, retries=np.array([0, 0, 2, 0], np.uint8), flags=np.zeros(4, np.uint8))
        t0 = int(time.time())
        r = q.drain("json_sum", 16)
        t1 = int(time.time()) + 1
        assert [s for _, s, _ in r.records()] == ["RETRY", "COMPLETE", "RETRY", "COMPLETE"] and q.depth() == 2
        w = q.wire_encode("ws", "stub-1")
        assert w.n == 2 and list(w.status) == [0, 0]
        for k, (i, want_retries) in enumerate(((0, 1), (2, 3))):
            rec = json.loads(w.result(k))
            assert bytes(w.task_ids[k]) == bytes(ids[i]) and rec["task_id"] == str(uuid.UUID(bytes=bytes(ids[i])))
            assert rec["retries"] == want_retries and t0 <= rec["timestamp"] <= t1
            assert rec["args"] == calls[i] and rec["kwargs"] == {}
        # cancel a re-pushed task by id: it leaves no record, the other comes back RETRY_LIMIT (its retries are now 3)
        marked, out = q.cancel(ids[[0]])
        assert marked == 1 and out[0] == L.CANCEL_MARKED
        r = q.drain("json_sum", 16)
        assert r.n_popped == 2 and [(bytes(t), s) for t, s, _ in r.records()] == [(bytes(ids[2]), "RETRY_LIMIT")]
        assert q.depth() == 0
    finally:
        q.close()


def test_small_ring_repush_wraps_bytes_and_slots():
    """4 KiB of ring, 16 slots: the window's segment is freed and the re-push lands at the ring's start behind the
    pending segment (a byte wrap); after a few rounds the slots wrap as well."""
    q = small_queue(ring_bytes=4096, ring_tasks=16)
    try:
        q.set_retry_policy([KeyError], 5)
        pad = "x" * 205                                                                  # 6 tasks: 1.5 KiB
        a = [sdk_put_payload({"p": pad, "k": i}) for i in range(6)]                      # KeyError: retried
        b = [sdk_put_payload({"p": pad, "values": [i]}) for i in range(6)]               # complete
        ida, idb = ids_for(6, 5), ids_for(6, 6)
        push(q, a, ida)
        push(q, b, idb)
        seen = []
        for _ in range(12):
            if q.depth() == 0:
                break
            r = q.drain("json_sum", 6)
            seen += r.records()
        want = oracle_answers(a + b, np.concatenate([ida, idb]), np.zeros(12, np.uint8), np.zeros(12, np.uint8), "json_sum", [KeyError], 5)
        assert seen == want and q.depth() == 0
    finally:
        q.close()


def test_exactly_full_ring_where_every_task_retries():
    q = small_queue(ring_bytes=4096, ring_tasks=16)
    try:
        q.set_retry_policy([KeyError], 2)
        fill = sdk_put_payload({"k": "y" * 221})
        assert len(fill) == 256
        payloads = [fill] * 16
        ids = ids_for(16, 8)
        push(q, payloads, ids)
        assert q.depth_bytes() == 4096 and q.depth() == 16
        with pytest.raises(L.B9Error):
            push(q, [b'{"args": [1], "kwargs": {}}'], ids_for(1, 9))            # the ring is full
        for want in ("RETRY", "RETRY", "RETRY_LIMIT"):
            r = q.drain("json_sum", 16)
            assert r.n == 16 and all(s == want for _, s, _ in r.records())
            assert [bytes(t) for t, _, _ in r.records()] == [bytes(i) for i in ids]
        assert q.depth() == 0
    finally:
        q.close()


@pytest.mark.parametrize("window", [1, 3, 5, 7, 12])
def test_exactly_full_ring_windows_ending_inside_push_segments(window):
    """A ring full in bytes and slots (two push segments, the first of 250-byte tasks so that task boundaries are not
    256-aligned), drained with windows that end inside a segment and whose every task retries: each fetch commits (the
    partly consumed segment gives its consumed bytes back), including re-pushes that straddle the ring's end, and the
    answers over all drains are the oracle's."""
    q = small_queue(ring_bytes=4096, ring_tasks=16)
    try:
        q.set_retry_policy([KeyError], 4)
        a = [sdk_put_payload({"k": "a%02d" % i + "y" * 212}) for i in range(8)]
        b = [sdk_put_payload({"k": "b%02d" % i + "y" * 218}) for i in range(8)]
        assert {len(p) for p in a} == {250} and {len(p) for p in b} == {256}
        ida, idb = ids_for(8, 90), ids_for(8, 91)
        push(q, a, ida)
        push(q, b, idb)
        assert q.depth() == 16 and q.depth_bytes() == 8 * 250 + 8 * 256
        with pytest.raises(L.B9Error):
            push(q, [sdk_put_payload({"k": 1})], ids_for(1, 92))          # full: no free slot
        got = drain_all(q, "json_sum", window)
        want = oracle_answers(a + b, np.concatenate([ida, idb]), np.zeros(16, np.uint8), np.zeros(16, np.uint8), "json_sum", [KeyError], 4)
        assert got == want and len(got) == 16 * 5
        push(q, a, ida)                                                    # the ring's bookkeeping is whole again
        push(q, b, idb)
        assert q.depth() == 16
        q.set_retry_policy([], 0)
        assert [s for _, s, _ in q.drain("json_sum", 16).records()] == ["ERROR"] * 16
    finally:
        q.close()


def test_repush_racing_a_producer_thread():
    """Producers push whole batches while drains re-push: no task is lost or duplicated, every batch stays in one piece
    and in order, and the answers are those of the oracle for the order the device settled on."""
    q = small_queue(ring_bytes=1 << 24, ring_tasks=1 << 14)
    try:
        q.set_retry_policy([KeyError, TypeError], 1)
        seed = [sdk_put_payload({"k": i}) if i % 3 else sdk_put_payload({"values": [i]}) for i in range(300)]
        seed_ids = ids_for(300, 20)
        push(q, seed, seed_ids)
        batches = [([sdk_put_payload({"values": [b, i]}) for i in range(50)], ids_for(50, 100 + b)) for b in range(40)]
        errors = []

        def producer():
            try:
                for p, i in batches:
                    push(q, p, i)
            except Exception as e:                                       # pragma: no cover - reported below
                errors.append(e)
        th = threading.Thread(target=producer)
        th.start()
        got = []
        while th.is_alive() or q.depth():
            if q.depth():
                got += q.drain("json_sum", 97).records()
        th.join()
        assert not errors
        got += drain_all(q, "json_sum", 97)
        count = {}
        for t, s, _ in got:
            count[bytes(t)] = count.get(bytes(t), 0) + 1
        for k in range(300):
            assert count[bytes(seed_ids[k])] == (2 if k % 3 else 1)
        pos = {}
        for n, (t, s, _) in enumerate(got):
            pos.setdefault(bytes(t), []).append(n)
        last = -1
        for p, ids in batches:
            where = [pos[bytes(i)][0] for i in ids]
            assert all(len(pos[bytes(i)]) == 1 for i in ids)
            assert where == list(range(where[0], where[0] + len(ids))) and where[0] > last      # contiguous, FIFO
            last = where[-1]
        assert all(s == "COMPLETE" for p, ids in batches for t, s, _ in got if bytes(t) in {bytes(i) for i in ids})
    finally:
        q.close()


def _records(r):
    return (r.task_ids.tobytes(), r.status.tobytes(), r.has_result.tobytes(), r.lengths.tobytes(), r.fifo_payload().tobytes(), r.n_popped)


@pytest.mark.parametrize("handler", HANDLERS)
def test_mask_zero_is_byte_equal_to_no_policy(handler):
    payloads, ids, flags, retries = build_corpus(handler, 30 + HANDLERS.index(handler))
    a, b = small_queue(), small_queue()
    try:
        b.set_retry_policy(list(EXC_BITS), 3)
        b.set_retry_policy([], 3)
        for q in (a, b):
            push(q, payloads, ids, flags, retries)
        assert _records(a.drain(handler, 1 << 12)) == _records(b.drain(handler, 1 << 12))
        assert a.depth() == b.depth() == 0
    finally:
        a.close(); b.close()


@pytest.mark.parametrize("handler", HANDLERS)
def test_peek_shows_retry_and_pushes_nothing(handler):
    payloads, ids, flags, retries = build_corpus(handler, 40 + HANDLERS.index(handler))
    q = small_queue()
    try:
        q.set_retry_policy(list(EXC_BITS), 1)
        push(q, payloads, ids, flags, retries)
        n = len(payloads)
        q.drain_launch(handler, n, peek=True)
        p1 = q.fetch()
        assert q.depth() == n and q.running() == 0
        want = oracle_answers(payloads, ids, flags, retries, handler, list(EXC_BITS), 1)[:n]
        assert p1.records() == want
        q.drain_launch(handler, n, peek=True)
        assert _records(q.fetch()) == _records(p1) and q.depth() == n
    finally:
        q.close()


def test_pickle_tasks_and_the_endpoint_drain_are_unchanged_by_a_policy():
    import cloudpickle
    calls = [([1], {}), (["a", "b"], {}), ([{}], {}), (["x"], {"k": 1}), ([{"values": [1]}], {})]
    pick = [cloudpickle.dumps({"args": a, "kwargs": k}) for a, k in calls]
    bodies = [json.dumps({"args": a, "kwargs": k}).encode() for a, k in calls] + [b'{"values": 3}', b"{}"]
    a, b = small_queue(), small_queue()
    try:
        b.set_retry_policy(list(EXC_BITS), 3)
        for handler in HANDLERS:
            for q in (a, b):
                push(q, pick, ids_for(len(pick), 50), flags=np.full(len(pick), L.TF_PICKLE, np.uint8))
            assert _records(a.drain(handler, 64, full_pickle=True)) == _records(b.drain(handler, 64, full_pickle=True))
            for q in (a, b):
                push(q, bodies, ids_for(len(bodies), 51), flags=np.full(len(bodies), L.TF_HTTP_BODY, np.uint8))
            ra, rb = a.drain(handler, 64, endpoint=True), b.drain(handler, 64, endpoint=True)
            assert _records(ra) == _records(rb) and L.ST_ERROR in set(rb.status.tolist())
            assert a.depth() == b.depth() == 0
    finally:
        a.close(); b.close()


def test_set_retry_policy_rejects_unknown_bits():
    q = small_queue()
    try:
        assert q._lib.b9_set_retry_policy(q._ctx, 0x40, 1) == L.B9_EINVAL
        assert q._lib.b9_set_retry_policy(None, 0x1, 1) == L.B9_EINVAL
        assert q._lib.b9_set_retry_policy(q._ctx, 0x1, 256) == L.B9_EINVAL     # a slot's retries is one byte
        assert q._lib.b9_set_retry_policy(q._ctx, 0x1, 255) == L.B9_OK
        assert STATUS_NAMES[L.ST_RETRY_LIMIT] == "RETRY_LIMIT"
    finally:
        q.close()


def test_sdk_mirror_retry_for_and_retries():
    from beta9_b200.taskqueue import TaskQueue
    tq = TaskQueue(retry_for=[KeyError], retries=2, gpu_handler="json_sum")
    q = small_queue()
    tq._queue = q
    try:
        @tq
        def json_sum(obj):
            return sum(obj["values"])
        t = json_sum.put({"no_values": [1]})
        ok = json_sum.put({"values": [1, 2]})
        got = json_sum.process_tasks()
        assert [(x.id, x.status) for x in got] == [(t.id, "RETRY"), (ok.id, "COMPLETE")] and got[1].result == 3
        assert [(x.id, x.status) for x in json_sum.process_tasks()] == [(t.id, "RETRY")]
        assert [(x.id, x.status) for x in json_sum.process_tasks()] == [(t.id, "RETRY_LIMIT")]
        assert json_sum.process_tasks() == [] and q.depth() == 0
        # a binascii.Error is not a ValueError to retry_for (exact class match)
        tq2 = TaskQueue(retry_for=[ValueError], retries=2, gpu_handler="vadd_f32", queue=q)

        @tq2
        def vadd(x):
            return x
        vadd.put("AAA*")
        vadd.put("AAAAAAAAAAAAAAAA")
        assert [x.status for x in vadd.process_tasks()] == ["ERROR", "RETRY"]
        assert binascii.Error is not ValueError
    finally:
        q.close()
