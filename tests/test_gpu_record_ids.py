"""GPU: every record's task id against the ids that were pushed.

A launch that leaves a record for every task of its window (nothing pending is cancelled, and always for the wire
encoder) does not copy ids: record j is the window's task j, and the fetch copies the ids straight from the window's
ring slots, in two pieces when the window wraps the slot ring. Count-mode launches (cancelled slots compacted away)
write the ids of their records as before. Checked here:
* dense windows that wrap the slot ring, for every handler, peek and non-peek;
* a burst of async peek launches followed by a push, then the fetch;
* a peek fetch followed by a non-peek drain of the same window;
* a fetch refused with B9_ENOSPC and retried;
* count mode (push flags, b9_cancel) and the switch back to dense windows;
* the endpoint drain in both modes; b9_wire_encode / _full; b9_drain_fetch_object;
* TaskMessage records whose bodies hold escapes the main loop does not settle (checked against their id in the
  kernel's tail), dense and in count mode."""
import ctypes as C
import json
import uuid

import numpy as np
import pytest

from beta9_b200 import _lib as L
from beta9_b200 import synth

pytestmark = pytest.mark.gpu
RING_TASKS = 1 << 12


def small_queue():
    from beta9_b200.device_queue import DeviceQueue
    return DeviceQueue(ring_bytes=1 << 24, ring_tasks=RING_TASKS, max_drain_tasks=RING_TASKS, max_result_bytes=1 << 24)


@pytest.fixture
def q():
    dq = small_queue()
    yield dq
    dq.close()


def move_head(q, k: int, seed: int) -> None:
    """push and drain k filler tasks, so that the next window starts at slot k % RING_TASKS"""
    assert q.depth() == 0
    b = synth.strings_batch(k, 16, seed=seed)
    q.push_batch(b.task_ids, b.payload, b.offsets)
    r = q.drain("identity", max_tasks=k)
    assert r.n == k and np.array_equal(r.task_ids, b.task_ids)


def make_batch(handler: str, n: int, seed: int) -> synth.Batch:
    if handler == "identity":
        return synth.strings_batch(n, 64, adversarial_frac=0.05, seed=seed)
    if handler == "crc32":
        return synth.crc_batch(n, seed=seed, lengths=np.full(n, 100, np.int64))
    if handler == "vadd_f32":
        return synth.vadd_batch(n, seed=seed)
    return synth.json_batch(n, doc_bytes=256, seed=seed)


def peek(q, handler, n, endpoint=False):
    q.drain_launch(handler, n, peek=True, endpoint=endpoint)
    return q.fetch()


@pytest.mark.parametrize("handler", ["identity", "crc32", "vadd_f32", "json_sum"])
def test_dense_window_wrapping_the_ring(q, handler):
    move_head(q, 3000, seed=11)
    b = make_batch(handler, 2000, seed=12)                # slots 3000 .. 4999: the window wraps at 4096
    q.push_batch(b.task_ids, b.payload, b.offsets)
    p = peek(q, handler, b.n)
    assert p.n == b.n and np.array_equal(p.task_ids, b.task_ids)
    part = peek(q, handler, 1000)                         # the part before the wrap: one piece
    assert part.n == 1000 and np.array_equal(part.task_ids, b.task_ids[:1000])
    r = q.drain(handler, max_tasks=b.n)
    assert r.n == b.n and q.depth() == 0 and np.array_equal(r.task_ids, b.task_ids)
    assert np.array_equal(r.status, p.status) and np.array_equal(r.fifo_payload(), p.fifo_payload())


def test_window_ending_at_the_last_slot(q):
    move_head(q, RING_TASKS - 500, seed=13)
    b = synth.strings_batch(700, 32, seed=14)
    q.push_batch(b.task_ids, b.payload, b.offsets)
    r = q.drain("identity", max_tasks=500)                # exactly up to the ring's end: one piece
    assert r.n == 500 and np.array_equal(r.task_ids, b.task_ids[:500])
    r = q.drain("identity")                               # from slot 0
    assert r.n == 200 and np.array_equal(r.task_ids, b.task_ids[500:])


def test_async_peek_burst_then_push_then_fetch(q):
    move_head(q, 3500, seed=15)
    b1 = synth.strings_batch(1500, 64, adversarial_frac=0.05, seed=16)
    b2 = synth.strings_batch(900, 64, seed=17)
    q.push_batch(b1.task_ids, b1.payload, b1.offsets)
    for m in (1500, 400, 1200):                           # the records waiting are the last launch's
        assert q.drain_launch("identity", m, peek=True, wait=False) == m
    q.push_batch(b2.task_ids, b2.payload, b2.offsets)
    r = q.fetch()
    assert r.n == 1200 and np.array_equal(r.task_ids, b1.task_ids[:1200])
    r = q.drain("identity", max_tasks=RING_TASKS)
    assert r.n == 2400 and np.array_equal(r.task_ids, np.concatenate([b1.task_ids, b2.task_ids]))


def test_peek_fetch_then_non_peek_drain(q):
    move_head(q, 2500, seed=18)
    b = synth.strings_batch(2500, 48, adversarial_frac=0.05, seed=19)
    q.push_batch(b.task_ids, b.payload, b.offsets)
    p = peek(q, "identity", b.n)
    assert np.array_equal(p.task_ids, b.task_ids) and q.depth() == b.n
    r = q.drain("identity", max_tasks=1800)
    assert r.n == 1800 and np.array_equal(r.task_ids, b.task_ids[:1800])
    r = q.drain("identity")
    assert r.n == 700 and np.array_equal(r.task_ids, b.task_ids[1800:]) and q.depth() == 0


def test_fetch_refused_then_retried(q):
    move_head(q, 3800, seed=20)
    b = synth.strings_batch(1000, 64, seed=21)
    q.push_batch(b.task_ids, b.payload, b.offsets)
    q.drain_launch("identity", b.n)
    with pytest.raises(L.B9Error) as e:
        q._fetch(None, 1)                                 # too few result bytes: nothing is consumed
    assert e.value.code == L.B9_ENOSPC and q.depth() == b.n
    r = q.fetch()
    assert r.n == b.n and np.array_equal(r.task_ids, b.task_ids) and q.depth() == 0


def test_count_mode_and_back(q):
    move_head(q, 3300, seed=22)
    b = synth.strings_batch(2000, 64, adversarial_frac=0.05, seed=23)
    cancelled = np.random.default_rng(24).random(b.n) < 0.1
    q.push_batch(b.task_ids, b.payload, b.offsets, flags=cancelled.astype(np.uint8) * L.TF_CANCELLED)
    p = peek(q, "identity", b.n)
    assert p.n == b.n - cancelled.sum() and np.array_equal(p.task_ids, b.task_ids[~cancelled])
    r = q.drain("identity", max_tasks=b.n)
    assert np.array_equal(r.task_ids, b.task_ids[~cancelled]) and q.depth() == 0
    # cancelled by id while pending, then a dense window again once they are drained
    b2 = synth.strings_batch(1500, 64, seed=25)
    q.push_batch(b2.task_ids, b2.payload, b2.offsets)
    marked, _ = q.cancel(b2.task_ids[::7])
    assert marked == len(b2.task_ids[::7])
    keep = np.ones(b2.n, bool)
    keep[::7] = False
    r = q.drain("crc32", max_tasks=b2.n)
    assert np.array_equal(r.task_ids, b2.task_ids[keep])
    b3 = synth.strings_batch(1500, 64, seed=26)
    q.push_batch(b3.task_ids, b3.payload, b3.offsets)
    r = q.drain("identity")
    assert r.n == b3.n and np.array_equal(r.task_ids, b3.task_ids)


def test_endpoint_drain_dense_and_count_mode(q):
    move_head(q, 3400, seed=27)
    bodies = [json.dumps({"x": i, "s": "a" * (i % 50)}).encode() for i in range(1500)]
    b = synth.from_payloads(bodies, seed=28)
    q.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, L.TF_HTTP_BODY, np.uint8))
    p = peek(q, "identity", b.n, endpoint=True)
    assert p.n == b.n and np.array_equal(p.task_ids, b.task_ids)
    r = q.drain("identity", max_tasks=b.n, endpoint=True)
    assert np.array_equal(r.task_ids, b.task_ids) and np.array_equal(r.fifo_payload(), p.fifo_payload())
    b2 = synth.from_payloads(bodies, seed=29)
    cancelled = np.random.default_rng(30).random(b2.n) < 0.2
    q.push_batch(b2.task_ids, b2.payload, b2.offsets,
                 flags=(L.TF_HTTP_BODY | cancelled.astype(np.uint8) * L.TF_CANCELLED).astype(np.uint8))
    p = peek(q, "json_sum", b2.n, endpoint=True)
    assert np.array_equal(p.task_ids, b2.task_ids[~cancelled])
    r = q.drain("json_sum", max_tasks=b2.n, endpoint=True)
    assert np.array_equal(r.task_ids, b2.task_ids[~cancelled]) and q.depth() == 0


@pytest.mark.parametrize("full", [False, True])
def test_wire_encode_records(q, full):
    move_head(q, 3600, seed=31)
    b = synth.strings_batch(1200, 64, adversarial_frac=0.05, seed=32)
    cancelled = np.zeros(b.n, bool)
    cancelled[5::11] = True                               # a wire record for every pending slot, cancelled or not
    q.push_batch(b.task_ids, b.payload, b.offsets, flags=cancelled.astype(np.uint8) * L.TF_CANCELLED)
    w = q.wire_encode("ws", "stub", full=full)
    assert w.n == b.n and np.array_equal(w.task_ids, b.task_ids)
    ok = np.flatnonzero(w.status == 0)
    assert ok.size > 0.9 * b.n
    for i in ok[:50]:
        assert json.loads(w.result(int(i)))["task_id"] == str(uuid.UUID(bytes=b.task_ids[i].tobytes()))
    r = q.drain("identity")
    assert np.array_equal(r.task_ids, b.task_ids[~cancelled]) and q.depth() == 0


def test_drain_fetch_object(q):
    move_head(q, 3700, seed=33)
    b = synth.strings_batch(1000, 40, adversarial_frac=0.1, seed=34)
    q.push_batch(b.task_ids, b.payload, b.offsets)
    obj = q.drain_object("identity")
    rec = L.SinkRecord()
    lib = L.load()
    for i in range(b.n):
        assert lib.b9_sink_get(obj.ctypes.data, obj.size, i, C.byref(rec)) == 0
        assert C.string_at(rec.task_id, 16) == b.task_ids[i].tobytes(), i
    assert q.depth() == 0


def test_task_message_records_through_the_kernel_tail():
    """Go writes '<', '>' and '&' as \\u escapes that json.dumps does not: such records are settled in the kernel's tail,
    which checks the record's id text against the task's id. Dense and count-mode windows, on a wrapping ring."""
    from beta9_b200.device_queue import DeviceQueue
    strs = ["a<b", "x & y", "<>" * 40, "caf\u00e9 <3", "\u2028line", "plain", "q\"uote\\", "tab\tand<"] * 40
    b = synth.from_payloads([json.dumps({"args": (s,), "kwargs": {}}).encode() for s in strs], seed=35)
    with small_queue() as q, DeviceQueue(ring_bytes=1 << 24, ring_tasks=1 << 12, max_drain_tasks=1 << 12,
                                         max_result_bytes=1 << 24) as ref_q:
        ref_q.push_batch(b.task_ids, b.payload, b.offsets)
        w = ref_q.wire_encode("ws", "stub")
        want = ref_q.drain("identity")                    # what the payloads themselves drain to
        enc = np.flatnonzero(w.status == 0)
        assert enc.size > 0.9 * b.n
        recs = [w.result(int(i)) for i in enc]
        off = np.zeros(enc.size + 1, np.uint64)
        np.cumsum([len(x) for x in recs], out=off[1:])
        pl = np.frombuffer(b"".join(recs), np.uint8)
        for cancelled in (np.zeros(enc.size, bool), np.arange(enc.size) % 5 == 2):
            move_head(q, 3900, seed=36)
            q.push_batch(b.task_ids[enc], pl, off, flags=(L.TF_TASK_MSG | cancelled.astype(np.uint8) * L.TF_CANCELLED).astype(np.uint8))
            r = q.drain("identity")
            keep = enc[~cancelled]
            assert r.n == keep.size and np.array_equal(r.task_ids, b.task_ids[keep])
            assert np.array_equal(r.status, want.status[keep]) and np.array_equal(r.has_result, want.has_result[keep])
            assert all(r.result(j) == want.result(int(i)) for j, i in enumerate(keep))
