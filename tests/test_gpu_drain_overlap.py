"""GPU: back-to-back drains overlap (programmatic dependent launch) and share a ring of control blocks that the kernels
zero for each other. A burst of B9_DRAIN_ASYNC peek drains must leave, in its last launch, exactly the records a blocking
b9_drain of the same window gives: status, has_result, id and result bytes, in FIFO order — for every handler, for the
tasks that go to the identity kernel's tail, across handler switches, around b9_cancel / b9_expire (count mode), after an
overflow, and around b9_wire_encode."""
import time

import numpy as np
import pytest

from beta9_b200 import synth
from beta9_b200._lib import B9_ENOSPC, TF_HTTP_BODY, TF_PICKLE, TF_TASK_MSG, B9Error
from oracle.pyoracle import funcloop, loop

pytestmark = pytest.mark.gpu
HANDLERS = ["identity", "crc32", "vadd_f32", "json_sum"]


@pytest.fixture(scope="module")
def dq():
    from beta9_b200.device_queue import DeviceQueue
    q = DeviceQueue(ring_bytes=1 << 31, ring_tasks=1 << 22, max_drain_tasks=1 << 21, max_result_bytes=1 << 30)
    yield q
    q.close()


def same_records(a, b, where=""):
    assert a.n == b.n, (where, a.n, b.n)
    assert np.array_equal(a.task_ids, b.task_ids), where
    bad = np.flatnonzero((a.status != b.status) | (a.has_result != b.has_result) | (a.lengths != b.lengths))
    assert bad.size == 0, (where, bad[:5])
    assert np.array_equal(a.fifo_payload(), b.fifo_payload()), where


def burst(q, handlers, sizes):
    """async peek drains back to back; the records of the last one"""
    for h, m in zip(handlers, sizes):
        assert q.drain_launch(h, m, peek=True, wait=False) == min(m, q.depth())
    return q.fetch()


def check_burst(q, b, handlers, sizes, flags=None, where=""):
    """push b, run the burst, then compare its last launch with a blocking drain of the same window; empties the queue"""
    assert q.depth() == 0
    q.push_batch(b.task_ids, b.payload, b.offsets, flags=flags)
    got = burst(q, handlers, sizes)
    want = q.drain(handlers[-1], sizes[-1])
    same_records(got, want, where)
    if q.depth():
        q.drain("identity")
    assert q.depth() == 0
    return got


def tail_batch(seed: int):
    """tasks the identity main loop defers or settles off its fast path: non-canonical escapes, HTTP bodies, pickles,
    TaskMessage records, between SDK strings with escapes"""
    rng = np.random.default_rng(seed)
    s = synth.strings_batch(3_000, 120, adversarial_frac=0.2, seed=seed)
    ids = [bytes(s.task_ids[i]) for i in range(s.n)]
    live = loop.run_task_loop(s.tasks(), ids, "identity", keep_wire=True)
    odd = [b'{"args": ["\\u0041b\\/c"], "kwargs": {}}', b'{"args": ["x\\u00e9\\ud83d\\ude00"], "kwargs": {}}',
           b'{"kwargs": {}, "args": ["swapped"]}', b'{"args": ["a\\tb"], "kwargs": {}}']
    blobs, flags = [], []
    for i in range(s.n):
        k = int(rng.integers(0, 10))
        if k < 4:
            blobs.append(s.task(i)); flags.append(0)
        elif k < 6:
            blobs.append(live[i].wire); flags.append(TF_TASK_MSG)
        elif k == 6:
            blobs.append(s.task(i)); flags.append(TF_HTTP_BODY)
        elif k == 7:
            blobs.append(funcloop.frame_map_input("y" * int(rng.integers(0, 60)))); flags.append(TF_PICKLE)
        else:
            blobs.append(odd[k - 8 + 2 * int(rng.integers(0, 2))]); flags.append(0)
    return synth.from_payloads(blobs, seed=seed), np.array(flags, np.uint8)


def handler_batch(handler: str, seed: int):
    if handler == "identity":
        return synth.strings_batch(100_000, 256, adversarial_frac=0.01, seed=seed)
    if handler == "crc32":
        return synth.crc_batch(50_000, seed=seed)
    if handler == "vadd_f32":
        return synth.vadd_batch(200_000, seed=seed)
    return synth.json_batch(25_000, seed=seed)


@pytest.mark.parametrize("k", [2, 5, 20])
def test_configs1_identity_burst(dq, k):
    b = synth.strings_batch(1_000_000, 256, adversarial_frac=0.01, seed=7 + k)
    check_burst(dq, b, ["identity"] * k, [b.n] * k, where=k)


@pytest.mark.parametrize("handler", HANDLERS)
@pytest.mark.parametrize("k", [2, 7])
def test_burst_per_handler(dq, handler, k):
    """windows of different sizes inside the burst: every launch sizes its grid and control block use anew"""
    b = handler_batch(handler, 100 + k)
    rng = np.random.default_rng(k)
    sizes = [int(x) for x in rng.integers(1, b.n + 1, k - 1)] + [b.n]
    check_burst(dq, b, [handler] * k, sizes, where=(handler, k))


@pytest.mark.parametrize("handler", HANDLERS)
def test_burst_of_tail_tasks(dq, handler):
    b, flags = tail_batch(31)
    check_burst(dq, b, [handler] * 4, [b.n] * 4, flags=flags, where=handler)


def test_burst_switching_handlers(dq):
    b = synth.concat([synth.strings_batch(20_000, 200, seed=41), synth.crc_batch(5_000, seed=42),
                      synth.vadd_batch(20_000, seed=43), synth.json_batch(3_000, seed=44)])
    seq = ["identity", "crc32", "vadd_f32", "json_sum", "identity", "json_sum", "crc32", "crc32", "vadd_f32", "identity"]
    for end in range(1, len(seq)):            # every handler follows every other one at least once, and itself
        check_burst(dq, b, seq[:end + 1], [b.n] * (end + 1), where=seq[:end + 1])


def keep_records(ref, keep):
    """the records of `ref` (a drain of the whole window) that belong to the tasks `keep`"""
    return ref.task_ids[keep], ref.status[keep], ref.has_result[keep], ref.lengths[keep], [ref.result(int(i)) for i in keep]


def assert_kept(r, ref, keep, where):
    ids, st, has, ln, res = keep_records(ref, keep)
    assert r.n == keep.size and np.array_equal(r.task_ids, ids), where
    assert np.array_equal(r.status, st) and np.array_equal(r.has_result, has) and np.array_equal(r.lengths, ln), where
    assert all(r.result(j) == res[j] for j in range(r.n)), where


@pytest.mark.parametrize("handler", ["identity", "json_sum"])
def test_burst_then_cancel_then_count_mode_drain(dq, handler):
    b = handler_batch(handler, 51)
    dq.push_batch(b.task_ids, b.payload, b.offsets)
    ref = burst(dq, [handler] * 3, [b.n] * 3)
    gone = np.sort(np.random.default_rng(52).choice(b.n, b.n // 10, replace=False))
    marked, _ = dq.cancel(b.task_ids[gone])
    assert marked == gone.size
    burst(dq, [handler] * 3, [b.n] * 3)       # count mode: the count kernels run between these launches
    r = dq.drain(handler, b.n)
    assert r.n_popped == b.n and dq.depth() == 0
    assert_kept(r, ref, np.setdiff1d(np.arange(b.n), gone), handler)


def test_burst_then_expire_then_count_mode_drain(dq):
    b = handler_batch("identity", 61)
    exp = np.zeros(b.n, np.int64)
    old = np.sort(np.random.default_rng(62).choice(b.n, b.n // 20, replace=False))
    exp[old] = 1                                # long past
    exp[exp == 0] = time.time_ns() + 3600 * 10**9
    dq.push_batch(b.task_ids, b.payload, b.offsets, expires_unix_ns=exp)
    ref = burst(dq, ["identity"] * 4, [b.n] * 4)
    assert dq.expire(time.time_ns()) == old.size
    r = dq.drain("identity", b.n)
    assert r.n_popped == b.n and dq.depth() == 0
    assert_kept(r, ref, np.setdiff1d(np.arange(b.n), old), "expire")


def test_burst_whose_last_launch_overflows():
    from beta9_b200.device_queue import DeviceQueue
    b = synth.strings_batch(40_000, 256, seed=71)             # ~10 MB of results
    with DeviceQueue(ring_bytes=1 << 26, ring_tasks=1 << 17, max_drain_tasks=1 << 17, max_result_bytes=4 << 20) as q:
        q.push_batch(b.task_ids, b.payload, b.offsets)
        for h in ("identity", "identity", "crc32"):
            q.drain_launch(h, 5_000, peek=True, wait=False)
        q.drain_launch("identity", b.n, peek=True, wait=False)
        with pytest.raises(B9Error) as e:
            q.sync()
        assert e.value.code == B9_ENOSPC
        assert q.depth() == b.n
        got = burst(q, ["identity"] * 3, [10_000] * 3)          # the next drains start from a clean control block
        want = q.drain("identity", 10_000)
        same_records(got, want, "after overflow")


def test_more_launches_than_control_blocks_then_wire_encode(dq):
    b = handler_batch("identity", 81)
    dq.push_batch(b.task_ids, b.payload, b.offsets)
    burst(dq, ["identity", "crc32", "identity", "json_sum", "identity"], [b.n] * 5)
    w = dq.wire_encode("ws", "stub", max_tasks=b.n // 2)
    assert w.n == b.n // 2 and dq.depth() == b.n
    got = burst(dq, ["identity"] * 3, [b.n] * 3)   # the encoder used the control ring: the launches after it start clean
    same_records(got, dq.drain("identity", b.n), "after wire_encode")
    assert dq.depth() == 0
