"""The queue model (tests/queue_model.py) pinned on the CPU: drained one window at a time it gives the oracle loops'
answers, its cancel and expire rules give the outcomes the library documents, and its operation generator is
deterministic for a seed."""
import json
import uuid

import pytest

from oracle.pyoracle import callback as CB
from oracle.pyoracle.loop import run_task_loop
from tests import queue_model as QM
from tests.golden.make_ref_callback_golden import explicit_wires
from tests.golden.make_ref_retry_golden import corpus_wires
from tests.retry_oracle import run_retry_loop


def drain_all(m, handler, window):
    out = []
    while m.depth():
        m.launch(handler, window)
        out += [(r.id, r.status, r.result) for r in m.fetch().records]
    return out


@pytest.mark.parametrize("handler", QM.HANDLERS)
@pytest.mark.parametrize("window", [1, 7, 1000])
def test_plain_loop_equals_run_task_loop(handler, window):
    items = [it for it in QM.corpus() if it.flags == 0]
    ids = [QM.task_id(3, k) for k in range(len(items))]
    m = QM.QueueModel(1 << 20, 1 << 12)
    m.push([QM.Task(i, it.payload) for i, it in zip(ids, items)])
    want = run_task_loop([it.payload for it in items], ids, handler)
    assert drain_all(m, handler, window) == [(w.task_id, w.status, w.result) for w in want]
    assert m.depth() == 0 and m.tasks_drained == len(items)


@pytest.mark.parametrize("handler", QM.HANDLERS)
@pytest.mark.parametrize("classes,max_retries", [((), 0), ((KeyError,), 2), ((TypeError, ValueError), 1), (tuple(QM.RETRY_CLASSES), 3)])
def test_retry_loop_on_the_golden_records(handler, classes, max_retries):
    wires = corpus_wires(handler) + explicit_wires(handler)
    ids = [uuid.UUID(json.loads(w)["task_id"]).bytes for w in wires]
    retries = [k % 3 for k in range(len(wires))]
    m = QM.QueueModel(1 << 24, 1 << 14)
    m.set_retry_policy(classes, max_retries)
    m.push([QM.Task(i, w, QM.TF_TASK_MSG, r) for i, w, r in zip(ids, wires, retries)])
    want = run_retry_loop(wires, ids, handler, retry_for=classes, max_retries=max_retries, retries=retries, task_msg=[True] * len(wires))
    assert drain_all(m, handler, 97) == [(a.task_id, a.status, a.result) for a in want]
    assert m.depth() == 0


def test_callback_kinds_of_retried_records_are_none():
    m = QM.QueueModel(1 << 16, 64)
    m.set_retry_policy([KeyError], 1)
    m.set_callback_policy(b"k")
    m.push([QM.Task(QM.task_id(4, 0), b'{"args": [{}], "kwargs": {}}'), QM.Task(QM.task_id(4, 1), b'{"args": [{}], "kwargs": {}}', retries=1),
            QM.Task(QM.task_id(4, 2), b"not json"), QM.Task(QM.task_id(4, 3), b'{"args": [{"values": [1]}], "kwargs": {}}')])
    w = m.launch("json_sum", 16)
    assert [(r.status, r.kind) for r in w.records] == [("RETRY", CB.CB_NONE), ("RETRY_LIMIT", CB.CB_NONE), ("REJECTED", CB.CB_NONE),
                                                       ("COMPLETE", CB.CB_POST)]
    assert QM.expected_digest(w.records[0], b"k", 1) == bytes(32) and QM.expected_digest(w.records[3], b"k", 1) != bytes(32)


def test_scripted_cancel_and_expire():
    m = QM.QueueModel(1 << 16, 64)
    ids = [QM.task_id(5, k) for k in range(8)]
    p = b'{"args": ["x"], "kwargs": {}}'
    m.push([QM.Task(ids[0], p, QM.TF_CANCELLED), QM.Task(ids[1], p, expires=100), QM.Task(ids[2], p, expires=300),
            QM.Task(ids[3], p), QM.Task(ids[4], p), QM.Task(ids[3], p)])
    assert m.expire(0) == 0 and m.expire(99) == 0
    assert m.expire(100) == 1 and m.expire(100) == 0                              # 0 < expires <= now, once
    marked, out = m.cancel([ids[0], ids[1], ids[3], ids[7], ids[3]])
    assert marked == 2 and out == [QM.ALREADY, QM.ALREADY, QM.MARKED, 0, QM.MARKED]  # an id on two slots: both marked
    w = m.launch("identity", 4)                                                  # claims ids 0-3
    assert m.running() == 4 and [r.id for r in w.records] == [ids[2]]
    marked, out = m.cancel([ids[2], ids[4], ids[3]])
    assert marked == 1 and out == [QM.CLAIMED, QM.MARKED, QM.CLAIMED | QM.ALREADY]
    assert m.expire(1000) == 1                                                   # the sweep covers the claimed window
    with pytest.raises(QM.ModelError) as e:
        m.fetch(too_small=True)
    assert e.value.code == QM.B9_ENOSPC and m.running() == 4 and m.depth() == 6
    assert m.fetch().records == w.records and m.depth() == 2 and m.running() == 0
    with pytest.raises(QM.ModelError):
        m.fetch()                                                                # committed exactly once
    m.launch("identity", 8, peek=True)                                           # a peek consumes nothing and claims nothing
    assert m.running() == 0 and m.cancel([ids[4]]) == (0, [QM.ALREADY])
    assert m.fetch().n == 2 and m.depth() == 2


def test_retry_after_expire_in_the_claimed_window():
    """The re-push carries the flags the task was pushed with, its retries + 1 and the same expiry: the next expire
    cancels it, and until then it drains again."""
    m = QM.QueueModel(1 << 16, 64)
    m.set_retry_policy([KeyError], 3)
    t = QM.Task(QM.task_id(6, 0), b'{"args": [{}], "kwargs": {}}', retries=1, expires=500)
    m.push([t])
    m.launch("json_sum", 8)
    assert m.expire(600) == 1
    w = m.fetch(now_s=(10, 11))
    assert [r.status for r in w.records] == ["RETRY"]
    (again,) = m.pending
    assert (again.id, again.payload, again.flags, again.retries, again.expires, again.ts) == (t.id, t.payload, 0, 2, 500, (10, 11))
    m.launch("json_sum", 8, peek=True)
    assert [r.status for r in m.fetch().records] == ["RETRY"]
    assert m.expire(600) == 1 and m.launch("json_sum", 8).records == []


@pytest.mark.parametrize("tiny", [True, False])
def test_generator_is_deterministic_and_replays(tiny):
    items = QM.corpus()
    shape = (4096, 32) if tiny else (1 << 20, 4096)
    m1, log1 = QM.run_model(17, 200, *shape, tiny=tiny, items=items)
    m2, log2 = QM.run_model(17, 200, *shape, tiny=tiny, items=items)
    assert log1 == log2 and m1.snapshot() == m2.snapshot()
    assert json.loads(json.dumps(log1)) == log1                                 # the log is plain data
    m3 = QM.QueueModel(*shape, shape[1])
    for op in log1:
        try:
            QM.apply(m3, op, items)
        except QM.ModelError:
            pass
    assert m3.snapshot() == m1.snapshot()
    kinds = {op["op"] for op in log1}
    assert {"push_batch", "cancel", "expire", "launch", "fetch"} <= kinds
