"""GPU: B9_DRAIN_PICKLE_FULL — the function path for every handler over plain values, against the oracle's runner loop
(funcloop.run_function_task) and the reference's own function runner (tests/golden/ref_function_golden.json). Records
drain3_kernel settles are the same with and without the flag; a count-mode window (cancelled slots) keeps every record
index; overflow, bursts and a wrapping ring behave as for any drain."""
import base64
import json
import os

import numpy as np
import pytest

from beta9_b200 import synth
from oracle.pyoracle import funcloop
from tests import pickle_corpus as PC

pytestmark = pytest.mark.gpu
TF_CANCELLED, TF_PICKLE, TF_TASK_MSG = 0x01, 0x04, 0x08
OK, ERROR, UNSUPPORTED = 0, 1, 4
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_function_golden.json")
GOLDEN_FULL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_function_full_golden.json")


@pytest.fixture(scope="module")
def dq():
    from beta9_b200.device_queue import DeviceQueue
    q = DeviceQueue(ring_bytes=1 << 29, ring_tasks=1 << 19, max_drain_tasks=1 << 19, max_result_bytes=1 << 28)
    yield q
    q.close()


def oracle(blob, handler):
    st_, res = funcloop.run_function_task(blob, handler)
    return (OK, res) if st_ == funcloop.COMPLETE else (ERROR, None)


def push(dq, blobs, flags=None, seed=0):
    b = synth.from_payloads(blobs, seed=seed)
    dq.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, TF_PICKLE, np.uint8) if flags is None else flags)
    return b


def check(r, blobs, handler, rows=None):
    answered = 0
    for i, blob in enumerate(blobs):
        k = i if rows is None else rows[i]
        got = (int(r.status[k]), r.result(k))
        if got[0] == UNSUPPORTED:
            assert got[1] is None
            continue
        answered += 1
        assert got == oracle(blob, handler), (handler, blob[:100])
    return answered


@pytest.mark.parametrize("handler", PC.HANDLERS)
def test_goldens_and_corpus(dq, handler):
    blobs = [base64.b64decode(c["args_pickle"]) for c in json.load(open(GOLDEN))["cases"]]
    blobs += PC.structured_blobs()
    push(dq, blobs)
    r = dq.drain(handler, full_pickle=True)
    assert r.n == len(blobs)
    assert check(r, blobs, handler) > len(blobs) // 2
    for i, blob in enumerate(blobs):                               # every decline has a documented reason
        if r.status[i] == UNSUPPORTED:
            assert PC.declined(blob, handler), blob[:100]


@pytest.mark.parametrize("handler", PC.HANDLERS)
def test_reference_goldens(dq, handler):
    """the results the reference's own function runner recorded, for every handler each golden ran"""
    cases = [c for g in (GOLDEN, GOLDEN_FULL) for c in json.load(open(g))["cases"] if handler in c["results"]]
    blobs = [base64.b64decode(c["args_pickle"]) for c in cases]
    push(dq, blobs)
    r = dq.drain(handler, full_pickle=True)
    assert r.n == len(blobs) and len(blobs) > 0
    answered = 0
    for i, c in enumerate(cases):
        if r.status[i] == UNSUPPORTED:
            assert r.result(i) is None and PC.declined(blobs[i], handler), c["input_repr"]
            continue
        answered += 1
        want = c["results"][handler]
        assert (int(r.status[i]), r.result(i)) == ((OK, base64.b64decode(want["result_pickle"])) if want["ok"] else (ERROR, None)), c["input_repr"]
    assert answered >= len(cases) - 6, handler


def test_configs4_documents_at_size(dq):
    b = synth.function_docs_batch(100_000)
    dq.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, TF_PICKLE, np.uint8))
    r = dq.drain("json_sum", full_pickle=True)
    assert r.n == b.n and np.array_equal(r.task_ids, b.task_ids) and int((r.status != OK).sum()) == 0
    raw = b.payload.tobytes()
    for i in range(0, b.n, 499):
        assert (OK, r.result(i)) == oracle(raw[int(b.offsets[i]):int(b.offsets[i + 1])], "json_sum")


def test_mixed_values_at_size(dq):
    vb = synth.values_batch(200_000, seed=3)
    vraw = vb.payload.tobytes()
    blobs = [funcloop.frame_map_input(json.loads(vraw[int(vb.offsets[i]):int(vb.offsets[i + 1])])["args"][0]) for i in range(vb.n)]
    push(dq, blobs)
    r = dq.drain("identity", full_pickle=True)
    assert r.n == len(blobs)
    assert int((r.status == UNSUPPORTED).sum()) < len(blobs) // 100
    sample = list(range(0, len(blobs), 97))
    check(r, [blobs[i] for i in sample], "identity", rows=sample)


def test_flag_leaves_drain3_records_alone(dq):
    """everything drain3_kernel settles (JSON tasks, the one-str template) is the same with and without the flag"""
    json_tasks = synth.values_batch(2000, seed=9)
    raw = json_tasks.payload.tobytes()
    blobs = [raw[int(json_tasks.offsets[i]):int(json_tasks.offsets[i + 1])] for i in range(json_tasks.n)]
    strs = [funcloop.frame_map_input("s%d" % i) for i in range(500)]
    flags = np.array([0] * len(blobs) + [TF_PICKLE] * len(strs), np.uint8)
    for handler in PC.HANDLERS:
        outs = []
        for full in (False, True):
            push(dq, blobs + strs, flags=flags)
            outs.append(dq.drain(handler, full_pickle=full).records())
        for a, b in zip(*outs):
            if a[1] != "UNSUPPORTED":
                assert a == b


@pytest.mark.parametrize("tile", [4, 8])
def test_count_mode_window_mixes(dq, tile):
    """pickle, JSON, TaskMessage-flagged and cancelled slots in one window: every record keeps its index, under both of
    json_sum's tile sizes. launch_drain3 picks 4-task tiles when the window has fewer 8-task tiles than
    3 x (resident CTAs per SM) x D3_WARPS x SMs, else 8. An SM holds at most 64 resident warps, so a window of at least
    1536 x SMs tasks gets 8-task tiles, and one of at most 8 x (3 x SMs - 1) tasks gets 4-task tiles (>= 1 warp per SM)."""
    sm = int(dq.stats().sm_count)
    n_docs = 6 * sm if tile == 4 else (1536 * sm * 3) // 4 + 8   # the window holds n_docs + n_docs // 3 tasks
    docs = synth.function_docs_batch(n_docs, seed=5)
    draw = docs.payload.tobytes()
    pick = [draw[int(docs.offsets[i]):int(docs.offsets[i + 1])] for i in range(docs.n)]
    js = synth.json_batch(n_docs // 3, seed=6)
    jraw = js.payload.tobytes()
    jblobs = [jraw[int(js.offsets[i]):int(js.offsets[i + 1])] for i in range(js.n)]
    rng = np.random.default_rng(n_docs)
    window = n_docs + n_docs // 3
    assert (window <= 8 * (3 * sm - 1)) if tile == 4 else (window >= 1536 * sm)
    blobs, flags = [], []
    for i, p in enumerate(pick):
        blobs.append(p); flags.append(TF_PICKLE | (TF_CANCELLED if rng.random() < 0.1 else 0))
        if i < len(jblobs):
            blobs.append(jblobs[i]); flags.append(0 if rng.random() < 0.8 else TF_TASK_MSG)
    flags = np.array(flags, np.uint8)
    b = push(dq, blobs, flags=flags, seed=n_docs)
    r = dq.drain("json_sum", full_pickle=True)
    live = np.nonzero((flags & TF_CANCELLED) == 0)[0]
    assert r.n == live.size and np.array_equal(r.task_ids, b.task_ids[live])
    for row, i in enumerate(live):
        if flags[i] == TF_PICKLE:
            assert (int(r.status[row]), r.result(row)) == oracle(blobs[i], "json_sum")


def test_async_bursts(dq):
    blobs = PC.sdk_blobs(300)
    push(dq, blobs)
    for _ in range(5):
        dq.drain_launch("identity", peek=True, wait=False, full_pickle=True)
    r = dq.fetch()
    assert r.n == len(blobs)
    check(r, blobs, "identity")
    dq.drain("identity")                                          # consume


def test_overflow_consumes_nothing(dq):
    from beta9_b200 import _lib as L
    from beta9_b200.device_queue import DeviceQueue
    q = DeviceQueue(ring_bytes=1 << 24, ring_tasks=1 << 12, max_drain_tasks=1 << 12, max_result_bytes=4096)
    try:
        blobs = [funcloop.frame_call(list(range(300)))] * 8
        push(q, blobs)
        with pytest.raises(L.B9Error) as e:
            q.drain("identity", full_pickle=True)
        assert e.value.code == L.B9_ENOSPC and q.depth() == len(blobs)
        r = q.drain("identity")                                   # without the flag the records are small enough
        assert r.n == len(blobs) and all(s == UNSUPPORTED for s in r.status)
    finally:
        q.close()


def test_small_wrapping_ring():
    from beta9_b200.device_queue import DeviceQueue
    q = DeviceQueue(ring_bytes=1 << 16, ring_tasks=64, max_drain_tasks=64, max_result_bytes=1 << 20)
    try:
        vals = [i * 1000 for i in range(40)] + ["w%d" % i for i in range(40)] + [[i, str(i)] for i in range(40)]
        for k in range(0, len(vals), 24):
            blobs = [funcloop.frame_call(v) for v in vals[k:k + 24]]
            push(q, blobs, seed=k)
            r = q.drain("identity", full_pickle=True)
            assert r.n == len(blobs) and check(r, blobs, "identity") == len(blobs)
    finally:
        q.close()


def test_function_map_full_pickle(dq):
    from beta9_b200.function import function

    @function(queue=dq, gpu_handler="json_sum", full_pickle=True)
    def total(obj):
        return sum(obj["values"])
    xs = [{"values": [1, 2, 3]}, {"values": [0.5, 0.25]}, {"values": []}, {"nope": 1}]
    assert list(total.map(xs)) == [6, 0.75, 0, None]
    assert total.unsupported == []

    @function(queue=dq, full_pickle=True)
    def echo(x):
        return x
    ys = [5, None, {"k": (1, 2)}, b"raw", 1.5, ("two", "args")]
    assert list(echo.map(ys)) == [5, None, {"k": (1, 2)}, b"raw", 1.5, None]      # (a tuple is the argument list: ERROR)
    assert echo.remote({"a": [1]}) == {"a": [1]}
