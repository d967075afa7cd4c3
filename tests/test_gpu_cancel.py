"""GPU tests of b9_cancel: StopTasks (pkg/api/v1/task.go:333-398) for pending tasks, by id, on the device. A task cancelled
this way must drain exactly like one pushed with B9_TF_CANCELLED; a drain's claimed window is left alone and reported."""
import os
import subprocess
import sys
import uuid

import numpy as np
import pytest

from beta9_b200 import _lib as L
from beta9_b200 import synth
from oracle import coracle

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MARKED, ALREADY, CLAIMED = L.CANCEL_MARKED, L.CANCEL_ALREADY, L.CANCEL_CLAIMED


@pytest.fixture(scope="module")
def dq():
    from beta9_b200.device_queue import DeviceQueue
    q = DeviceQueue(ring_bytes=1 << 31, ring_tasks=1 << 22, max_drain_tasks=1 << 22, max_result_bytes=1 << 30)
    yield q
    q.close()


def oracle_bytes(o, keep):
    """The oracle's result bytes of tasks `keep`, back to back (what DrainResult.fifo_payload gives for them)."""
    ln = np.diff(o.offsets).astype(np.int64)[keep]
    if ln.sum() == 0:
        return np.empty(0, np.uint8)
    ends = np.cumsum(ln)
    rec = np.repeat(np.arange(keep.size), ln)
    idx = np.arange(int(ends[-1]), dtype=np.int64)
    return o.payload[o.offsets[:-1].astype(np.int64)[keep][rec] + idx - (ends - ln)[rec]]


def assert_survivors(r, b, o, keep):
    assert r.n == keep.size and np.array_equal(r.task_ids, b.task_ids[keep])
    assert np.array_equal(r.status, o.status[keep]) and np.array_equal(r.has_result, o.has[keep])
    assert np.array_equal(r.lengths.astype(np.int64), np.diff(o.offsets).astype(np.int64)[keep])
    assert np.array_equal(r.fifo_payload(), oracle_bytes(o, keep))


def test_cancel_configs1_size(dq):
    """configs[1] size: 1 M 256-char strings, a shuffled 10 % cancelled in one call with 1 k duplicate and 1 k unknown ids."""
    b = synth.strings_batch(1_000_000, 256, adversarial_frac=0.01)
    rng = np.random.default_rng(11)
    gone_idx = rng.choice(b.n, 100_000, replace=False)
    dup = rng.choice(gone_idx, 1000)
    req = np.concatenate([b.task_ids[gone_idx], b.task_ids[dup], synth.task_ids(1000, seed=12345)])
    want = np.concatenate([np.full(101_000, MARKED, np.uint8), np.zeros(1000, np.uint8)])
    perm = rng.permutation(req.shape[0])
    dq.push_batch(b.task_ids, b.payload, b.offsets)
    marked, out = dq.cancel(req[perm])
    assert marked == 100_000 and np.array_equal(out, want[perm])
    assert dq.depth() == b.n                                     # counted until a drain pops them
    r = dq.drain("identity", b.n)
    assert r.n_popped == b.n and r.n == 900_000 and dq.depth() == 0
    gone = np.zeros(b.n, bool); gone[gone_idx] = True
    o = coracle.run_batch(b.task_ids, b.payload, b.offsets, "identity", nthreads=8)
    assert_survivors(r, b, o, np.flatnonzero(~gone))


@pytest.mark.parametrize("handler,make", [("identity", lambda: synth.strings_batch(70_001, 48, adversarial_frac=0.02, seed=31)),
                                          ("crc32", lambda: synth.crc_batch(3001, seed=32)),
                                          ("vadd_f32", lambda: synth.vadd_batch(9007, seed=33)),
                                          ("json_sum", lambda: synth.json_batch(1203, doc_bytes=400, seed=34))])
def test_cancel_equals_push_flags_every_handler(dq, handler, make):
    """The cancel patterns of test_cancelled_slots_every_handler: flags at push and b9_cancel after it drain byte-identically."""
    b = make()
    rng = np.random.default_rng(b.n)
    patterns = [rng.random(b.n) < 0.07, np.arange(b.n) == b.n // 3, np.arange(b.n) != 5,
                (np.arange(b.n) // 97) % 3 == 0, np.arange(b.n) < 40, np.arange(b.n) >= b.n - 33]
    for gone in patterns:
        dq.push_batch(b.task_ids, b.payload, b.offsets, flags=gone.astype(np.uint8))
        a = dq.drain(handler)
        dq.push_batch(b.task_ids, b.payload, b.offsets)
        marked, out = dq.cancel(b.task_ids[gone])
        assert marked == int(gone.sum()) and np.all(out == MARKED)
        c = dq.drain(handler)
        assert c.n_popped == a.n_popped == b.n and dq.depth() == 0
        assert c.n == a.n == int((~gone).sum())
        assert np.array_equal(c.task_ids, a.task_ids) and np.array_equal(c.status, a.status)
        assert np.array_equal(c.has_result, a.has_result) and np.array_equal(c.lengths, a.lengths)
        assert np.array_equal(c.fifo_payload(), a.fifo_payload())


def test_claimed_window_is_left_alone(dq):
    b = synth.strings_batch(40_000, 64, seed=41)
    dq.push_batch(b.task_ids, b.payload, b.offsets)
    dq.drain_launch("identity", 10_000, wait=False)
    marked, out = dq.cancel(b.task_ids[5000:15000])
    assert marked == 5000
    assert np.all(out[:5000] == CLAIMED) and np.all(out[5000:] == MARKED)
    r = dq.fetch()
    assert r.n == 10_000 and np.array_equal(r.task_ids, b.task_ids[:10_000])
    rest = dq.drain("identity")
    assert rest.n_popped == 30_000 and rest.n == 25_000 and np.array_equal(rest.task_ids, b.task_ids[15_000:])
    # cancelled_pending stayed exact: nothing cancelled is pending, so a drain needs no count pre-pass (1 launch)
    dq.push_batch(b.task_ids[:1000], b.payload[:int(b.offsets[1000])], b.offsets[:1001])
    k0 = dq.stats().kernel_launches
    assert dq.drain("identity").n == 1000
    assert dq.stats().kernel_launches - k0 == 1


def test_already_cancelled_and_duplicate_slots(dq):
    b = synth.strings_batch(3000, 32, seed=42)
    flags = np.zeros(b.n, np.uint8); flags[:1000] = L.TF_CANCELLED
    exp = np.zeros(b.n, np.int64); exp[1000:2000] = 1000
    dq.push_batch(b.task_ids, b.payload, b.offsets, expires_unix_ns=exp, flags=flags)
    assert dq.expire(2000) == 1000
    k0 = dq.stats().kernel_launches
    marked, out = dq.cancel(b.task_ids[:2500])
    assert dq.stats().kernel_launches - k0 == 1
    assert marked == 500 and np.all(out[:2000] == ALREADY) and np.all(out[2000:] == MARKED)
    marked, out = dq.cancel(b.task_ids[:2500])
    assert marked == 0 and np.all(out == ALREADY)
    assert dq.depth() == b.n
    r = dq.drain("identity")
    assert r.n_popped == b.n and np.array_equal(r.task_ids, b.task_ids[2500:])
    # one id pushed twice, the first copy cancelled at push: both bits, one slot marked
    one = b.slice(0, 1)
    dq.push_batch(one.task_ids, one.payload, one.offsets, flags=np.ones(1, np.uint8))
    dq.push_batch(one.task_ids, one.payload, one.offsets)
    marked, out = dq.cancel(np.concatenate([one.task_ids, one.task_ids]))
    assert marked == 1 and list(out) == [MARKED | ALREADY] * 2
    r = dq.drain("identity")
    assert r.n == 0 and r.n_popped == 2 and dq.depth() == 0


def test_peek_records_are_unchanged(dq):
    b = synth.strings_batch(20_000, 64, adversarial_frac=0.05, seed=43)
    o = coracle.run_batch(b.task_ids, b.payload, b.offsets, "identity")
    dq.push_batch(b.task_ids, b.payload, b.offsets)
    dq.drain_launch("identity", b.n, peek=True, wait=False)
    gone = np.arange(b.n) % 3 == 0
    marked, out = dq.cancel(b.task_ids[gone])
    assert marked == int(gone.sum()) and np.all(out == MARKED)        # after a peek nothing is claimed
    p = dq.fetch()
    assert_survivors(p, b, o, np.arange(b.n))
    r = dq.drain("identity")
    assert r.n_popped == b.n and dq.depth() == 0
    assert_survivors(r, b, o, np.flatnonzero(~gone))


def test_small_ring_wraps_against_fifo_model():
    """A 4 Ki-slot ring: pushes, cancels and partial drains interleaved so that the pending window, and the ids a cancel
    hits, straddle the end of the slot ring and of the payload ring; every drain against a Python FIFO model."""
    from beta9_b200.device_queue import DeviceQueue
    src = synth.strings_batch(30_000, 24, adversarial_frac=0.05, seed=44)
    o = coracle.run_batch(src.task_ids, src.payload, src.offsets, "identity")
    rng = np.random.default_rng(44)
    q = DeviceQueue(ring_bytes=1 << 19, ring_tasks=1 << 12, max_drain_tasks=1 << 12, max_result_bytes=1 << 20)
    try:
        model = []                                     # [source index, cancelled]
        nxt = 0
        for _ in range(60):
            k = int(rng.integers(200, 900))
            if nxt + k <= src.n and len(model) + k <= 3000:
                part = src.slice(nxt, nxt + k)
                q.push_batch(part.task_ids, part.payload, part.offsets)
                model += [[i, False] for i in range(nxt, nxt + k)]
                nxt += k
            if model:
                pick = set(int(j) for j in rng.choice(len(model), min(len(model), int(rng.integers(1, 300))), replace=False))
                pick |= {0, len(model) - 1}
                pick = sorted(pick)
                req = np.concatenate([src.task_ids[[model[j][0] for j in pick]], synth.task_ids(5, seed=int(rng.integers(1 << 30)) + 1000)])
                want = [ALREADY if model[j][1] else MARKED for j in pick] + [0] * 5
                marked, out = q.cancel(req)
                assert list(out) == want and marked == want.count(MARKED)
                for j in pick:
                    model[j][1] = True
            m = int(rng.integers(0, len(model) + 1))
            r = q.drain("identity", max_tasks=m) if m else None
            if r is not None:
                taken, model = model[:m], model[m:]
                keep = np.array([i for i, c in taken if not c], np.int64)
                assert r.n_popped == m
                assert_survivors(r, src, o, keep)
            assert q.depth() == len(model)
        r = q.drain("identity")
        keep = np.array([i for i, c in model if not c], np.int64)
        assert r.n_popped == len(model)
        assert_survivors(r, src, o, keep)
        assert nxt > 2 * (1 << 12)                      # the slot ring wrapped at least twice
    finally:
        q.close()


def test_one_mebi_ids_over_four_mebi_tasks(dq):
    """n = 2^20 ids, mostly absent, over 4 Mi pending tasks: the fence narrows each search to 512 keys in global memory."""
    b = synth.strings_batch(1 << 22, 8, adversarial_frac=0, seed=45)
    rng = np.random.default_rng(45)
    present = rng.choice(b.n, 5000, replace=False)
    req = np.concatenate([b.task_ids[present], synth.task_ids((1 << 20) - 5000, seed=4545)])
    want = np.concatenate([np.full(5000, MARKED, np.uint8), np.zeros((1 << 20) - 5000, np.uint8)])
    perm = rng.permutation(req.shape[0])
    dq.push_batch(b.task_ids, b.payload, b.offsets)
    marked, out = dq.cancel(req[perm])
    assert marked == 5000 and np.array_equal(out, want[perm])
    r = dq.drain("identity", b.n)
    gone = np.zeros(b.n, bool); gone[present] = True
    assert r.n_popped == b.n and r.n == b.n - 5000 and np.array_equal(r.task_ids, b.task_ids[~gone])
    assert dq.depth() == 0


def test_arguments_and_empty_queue(dq):
    lib, ctx = L.load(), dq._ctx
    ids = synth.task_ids(4, seed=46)
    assert dq.depth() == 0
    marked, out = dq.cancel(ids)                                      # nothing pending: every id reports 0
    assert marked == 0 and list(out) == [0, 0, 0, 0]
    marked, out = dq.cancel(np.zeros((0, 16), np.uint8))
    assert marked == 0 and out.size == 0
    assert lib.b9_cancel(ctx, None, 0, None) == 0
    assert lib.b9_cancel(ctx, None, 3, None) == L.B9_EINVAL
    assert lib.b9_cancel(None, ids.ctypes.data, 4, None) == L.B9_EINVAL
    big = np.zeros(((1 << 20) + 1, 16), np.uint8)
    assert lib.b9_cancel(ctx, big.ctypes.data, (1 << 20) + 1, None) == L.B9_E2BIG
    b = synth.strings_batch(100, 16, seed=46)
    dq.push_batch(b.task_ids, b.payload, b.offsets)
    assert lib.b9_cancel(ctx, b.task_ids.ctypes.data, 40, None) == 40      # outcome = NULL
    r = dq.drain("identity")
    assert r.n_popped == 100 and np.array_equal(r.task_ids, b.task_ids[40:])


def test_submitted_task_is_pending_only_after_flush(dq):
    tid = synth.task_ids(1, seed=47)
    dq.submit(tid[0].tobytes(), b'{"args": ["x"], "kwargs": {}}')
    assert dq.buffered() == 1
    marked, out = dq.cancel(tid)
    assert marked == 0 and out[0] == 0
    assert dq.flush() == 1
    marked, out = dq.cancel(tid)
    assert marked == 1 and out[0] == MARKED
    r = dq.drain("identity")
    assert r.n == 0 and r.n_popped == 1 and dq.depth() == 0


def test_sdk_stop_tasks():
    from beta9_b200.device_queue import DeviceQueue
    from beta9_b200.taskqueue import TaskQueue
    q = DeviceQueue(ring_bytes=1 << 24, ring_tasks=1 << 14, max_drain_tasks=1 << 14, max_result_bytes=1 << 24)
    try:
        w = TaskQueue(max_pending_tasks=10_000, gpu_handler="identity", queue=q)(lambda s: s)
        tasks = w.put_batch([((f"s{i}",), {}) for i in range(100)])
        stop = [tasks[i].id for i in (0, 50, 99)]
        unknown = str(uuid.uuid4())
        assert w.stop_tasks(stop + [unknown, "not-a-uuid"]) == {**{t: "CANCELLED" for t in stop}, unknown: "NOT_FOUND", "not-a-uuid": "NOT_FOUND"}
        assert w.stop_tasks(stop[:1]) == {stop[0]: "ALREADY_CANCELLED"}
        got = w.process_tasks()
        live = [i for i in range(100) if i not in (0, 50, 99)]
        assert [t.id for t in got] == [tasks[i].id for i in live] and [t.result for t in got] == [f"s{i}" for i in live]
        # claimed by a drain in flight: left alone
        tasks = w.put_batch([((f"r{i}",), {}) for i in range(10)])
        q.drain_launch("identity", 5, wait=False)
        assert w.stop_tasks([tasks[1].id, tasks[7].id]) == {tasks[1].id: "RUNNING", tasks[7].id: "CANCELLED"}
        assert q.fetch().n == 5
        assert [t.result for t in w.process_tasks()] == ["r5", "r6", "r8", "r9"]
        # map(): a task stopped while it is pending yields None
        put = w.put_batch

        def put_then_stop(calls):
            ts = put(calls)
            assert w.stop_tasks([ts[1].id]) == {ts[1].id: "CANCELLED"}
            return ts
        w.put_batch = put_then_stop
        assert list(w.map(["x", "y", "z"])) == ["x", None, "z"]
        assert q.depth() == 0
    finally:
        q.close()


def test_multi_gpu_cancel_before_and_after_rebalance(tmp_path):
    world = min(L.load().b9_device_count(), 4)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "_gpu_cancel_multi_worker.py"), str(r), str(world), str(tmp_path)],
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(world)]
    outs = [p.communicate(timeout=600)[0] for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o
    res = [np.load(os.path.join(tmp_path, f"cancel_rank{r}.npz")) for r in range(world)]
    first = {x.tobytes() for x in res[0]["first"]}
    second = [x.tobytes() for x in res[0]["second"]]
    # every id of the second list is pending on exactly one rank: MARKED there, or ALREADY if the first cancel took it
    for j, t in enumerate(second):
        bits = [int(r["outcome2"][j]) for r in res]
        want = ALREADY if t in first else MARKED
        assert sorted(bits) == [0] * (world - 1) + [want], (t.hex(), bits)
    assert sum(int(r["marked2"]) for r in res) == len(set(second) - first)
    gone = first | set(second)
    want = {}
    for r in res:
        o = coracle.run_batch(r["before_ids"], r["before_payload"], r["before_offsets"], "identity")
        for i in range(len(r["before_ids"])):
            t = r["before_ids"][i].tobytes()
            if t not in gone:
                want[t] = (int(o.status[i]), o.result(i))
    got = {}
    for r in res:
        off = np.concatenate([[0], np.cumsum(r["lens"].astype(np.int64))])
        for i in range(len(r["status"])):
            got[r["ids"][i].tobytes()] = (int(r["status"][i]), r["payload"][off[i]:off[i + 1]].tobytes() if r["has"][i] else None)
    assert sum(len(r["status"]) for r in res) == len(got) == len(want) and got == want
