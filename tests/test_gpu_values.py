"""GPU: identity over numbers and nested lists / objects (synth.values_batch) and json_sum over float64 documents
(synth.json_float_batch), through the C ABI, against the oracles -- plus a batch that mixes them with configs[1]'s
strings, whose records must be exactly those of a strings-only drain."""
import numpy as np
import pytest

from beta9_b200 import synth
from oracle import coracle
from oracle.pyoracle import loop

pytestmark = pytest.mark.gpu
CODE = {"COMPLETE": 0, "ERROR": 1, "RETRY": 2, "REJECTED": 3}


@pytest.fixture(scope="module")
def dq():
    from beta9_b200.device_queue import DeviceQueue
    q = DeviceQueue(ring_bytes=1 << 30, ring_tasks=1 << 20, max_drain_tasks=1 << 20, max_result_bytes=1 << 30)
    yield q
    q.close()


def run_gpu(dq, batch, handler):
    assert dq.depth() == 0
    dq.push_batch(batch.task_ids, batch.payload, batch.offsets)
    r = dq.drain(handler, max_tasks=batch.n)
    assert dq.depth() == 0 and r.n_popped == batch.n and r.n == batch.n
    assert np.array_equal(r.task_ids, batch.task_ids)
    return r


def check_python_oracle(batch, r, idx, handler):
    payloads = [batch.task(int(i)) for i in idx]
    want = loop.run_task_loop(payloads, [bytes(batch.task_ids[int(i)]) for i in idx], handler)
    for i, w in zip(idx, want):
        assert int(r.status[i]) == CODE[w.status], (batch.task(int(i)), int(r.status[i]), w.status)
        assert r.result(int(i)) == w.result, (batch.task(int(i)), r.result(int(i)), w.result)


def test_identity_values_batch(dq):
    b = synth.values_batch(200_000, seed=21)
    r = run_gpu(dq, b, "identity")
    assert int((r.status == 4).sum()) == 0                       # the generator stays inside the device's domain
    o = coracle.run_batch(b.task_ids, b.payload, b.offsets, "identity")
    answered = np.flatnonzero(o.status != 4)                     # the C oracle: integer and container data
    assert answered.size > 20_000
    for i in answered:
        assert int(r.status[i]) == int(o.status[i]) and r.result(int(i)) == o.result(int(i)), b.task(int(i))
    floats = np.flatnonzero(o.status == 4)                       # float-bearing: the Python oracle
    assert floats.size >= 20_000
    check_python_oracle(b, r, floats[:: max(1, floats.size // 25_000)], "identity")


def test_json_sum_float_batch(dq):
    b = synth.json_float_batch(50_000, seed=22)
    r = run_gpu(dq, b, "json_sum")
    assert int((r.status == 4).sum()) == 0
    check_python_oracle(b, r, np.arange(b.n), "json_sum")


def test_mixed_with_configs1_strings(dq):
    s = synth.strings_batch(60_000, 256, seed=23)
    v = synth.values_batch(6_000, seed=24)
    rng = np.random.default_rng(25)
    order = rng.permutation(s.n + v.n)                           # interleave: value tasks inside string tiles
    both = synth.concat([s, v])
    mixed = synth.from_payloads([both.task(int(i)) for i in order])
    mixed.task_ids[:] = both.task_ids[order]
    r_s = run_gpu(dq, s, "identity")
    r_m = run_gpu(dq, mixed, "identity")
    assert int((r_m.status == 4).sum()) == 0
    pos = np.empty(order.size, np.int64)
    pos[order] = np.arange(order.size)
    for i in range(s.n):                                         # the strings' records: identical to the strings-only drain
        j = int(pos[i])
        assert int(r_m.status[j]) == int(r_s.status[i]) and r_m.result(j) == r_s.result(i), i
    o = coracle.run_batch(s.task_ids, s.payload, s.offsets, "identity")
    assert np.array_equal(r_s.fifo_payload(), o.payload)
    check_python_oracle(mixed, r_m, np.flatnonzero(order >= s.n)[:3000], "identity")
