"""GPU tests of b9_endpoint_drain_launch: HTTP request bodies answered on the device with the endpoint runner's response
bytes (JSONResponse), against the reference's golden (tests/golden/ref_endpoint_golden.json) and the oracle's endpoint
request (oracle/pyoracle/endpoint.py), plus the drain contract it shares with b9_drain_launch: cancelled slots, peek,
async bursts mixed with task-queue drains, overflow, a wrapping ring, the result-sink object and b9_submit."""
import ctypes as C
import json
import re
import threading
import uuid

import numpy as np
import pytest

from beta9_b200 import _lib as L
from beta9_b200 import synth
from oracle.pyoracle import endpoint as EP
from oracle.pyoracle.handlers import HANDLERS as PYH

pytestmark = pytest.mark.gpu
HANDLERS = ["identity", "crc32", "vadd_f32", "json_sum"]
STATUS = {L.ST_COMPLETE: EP.OK, L.ST_REJECTED: EP.BAD_REQUEST, L.ST_ERROR: EP.HANDLER_RAISED}


@pytest.fixture(scope="module")
def dq():
    from beta9_b200.device_queue import DeviceQueue
    q = DeviceQueue(ring_bytes=1 << 31, ring_tasks=1 << 22, max_drain_tasks=1 << 22, max_result_bytes=1 << 30)
    yield q
    q.close()


def push_bodies(q, bodies, flags=L.TF_HTTP_BODY, ids=None):
    b = synth.from_payloads(list(bodies))
    tid = b.task_ids if ids is None else ids
    q.push_batch(tid, b.payload, b.offsets, flags=np.full(b.n, flags, np.uint8))
    return tid


def peek(q, handler, n, endpoint):
    """one blocking B9_DRAIN_PEEK launch and its records (the tasks stay pending)"""
    q.drain_launch(handler, n, peek=True, endpoint=endpoint)
    return q.fetch()


def outcomes(r):
    """(outcome, bytes) per record, the oracle's spelling; UNSUPPORTED as ("UNSUPPORTED", None)"""
    out = []
    for i in range(r.n):
        st = int(r.status[i])
        if st == L.ST_COMPLETE:
            assert r.has_result[i] == 1
            out.append((EP.OK, r.result(i)))
        else:
            assert r.has_result[i] == 0
            out.append((STATUS.get(st, "UNSUPPORTED"), EP.INVALID_PAYLOAD_BODY if st == L.ST_REJECTED else None))
    return out


_SURROGATE_ESCAPE = re.compile(rb"\\u[dD][89a-fA-F]")


class _Fallback(Exception):
    pass


def _int_only(s):
    v = int(s)
    if abs(v) >= 2**53:
        raise _Fallback
    return v


def _no_float(s):
    raise _Fallback


def quick_oracle(body, handler):
    """The oracle's answer computed with the stdlib json where Go's decoding and CPython's provably agree (valid UTF-8, no
    surrogate escapes, ints below 2^53 and no floats, exactly "args" and an empty "kwargs"); the full oracle otherwise."""
    try:
        if _SURROGATE_ESCAPE.search(body):
            raise _Fallback
        doc = json.loads(body.decode("utf-8"), parse_int=_int_only, parse_float=_no_float, parse_constant=_no_float)
        if not isinstance(doc, dict) or set(doc) != {"args", "kwargs"} or not isinstance(doc["args"], list) or doc["kwargs"] != {}:
            raise _Fallback
    except (_Fallback, ValueError):
        return EP.run_endpoint_request(body, handler)
    try:
        result = PYH[handler](*doc["args"])
    except BaseException:
        return EP.HANDLER_RAISED, None
    try:
        return EP.OK, EP.render(result)
    except BaseException:
        return EP.RENDER_FAILED, None


def check_batch(dq, b, handler, sample=1000):
    """push the SDK-framed batch as HTTP bodies, endpoint-drain it, compare every record with the quick oracle (itself
    checked against the full oracle on `sample` bodies)"""
    bodies = b.tasks()
    rng = np.random.default_rng(5)
    for i in rng.choice(len(bodies), min(sample, len(bodies)), replace=False):
        assert quick_oracle(bodies[i], handler) == EP.run_endpoint_request(bodies[i], handler)
    dq.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, L.TF_HTTP_BODY, np.uint8))
    r = dq.drain(handler, b.n, endpoint=True)
    assert r.n == b.n and r.n_popped == b.n and np.array_equal(r.task_ids, b.task_ids)
    got = outcomes(r)
    bad = [i for i in range(b.n) if got[i] != quick_oracle(bodies[i], handler)]
    assert not bad, [(bodies[i][:100], got[i], quick_oracle(bodies[i], handler)) for i in bad[:3]]
    return r


@pytest.mark.parametrize("handler", HANDLERS)
def test_reference_golden_on_device(dq, handler):
    from tests.test_endpoint_on_host import _golden_want, declined, golden_cases
    cases = golden_cases()
    bodies = [b for b, _ in cases]
    tid = push_bodies(dq, bodies)
    r = dq.drain(handler, len(bodies), endpoint=True)
    assert r.n == len(bodies) and np.array_equal(r.task_ids, tid)
    for (b, res), got in zip(cases, outcomes(r)):
        if got[0] == "UNSUPPORTED":
            assert declined(b, handler), b[:120]
            continue
        assert got == _golden_want(res[handler]), (b[:120], got)


def test_configs1_bodies_identity(dq):
    """configs[1] shape: 1 M 256-character strings, 1 % with escapes and non-ASCII, as HTTP bodies"""
    check_batch(dq, synth.strings_batch(1_000_000, 256, adversarial_frac=0.01), "identity")


@pytest.mark.parametrize("handler,make", [
    ("crc32", lambda: synth.crc_batch(100_000)),
    ("vadd_f32", lambda: synth.vadd_batch(100_000, floats_per_vec=32)),
    ("json_sum", lambda: synth.json_batch(20_000, doc_bytes=512)),
])
def test_synthetic_batches(dq, handler, make):
    check_batch(dq, make(), handler, sample=300)


def test_cancelled_slots_are_compacted(dq):
    """count mode: a shuffled 10 % cancelled with b9_cancel; the survivors' records equal an uncancelled drain's"""
    b = synth.strings_batch(50_000, 64, adversarial_frac=0.05, seed=21)
    dq.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, L.TF_HTTP_BODY, np.uint8))
    full = outcomes(peek(dq, "identity", b.n, True))
    gone = np.random.default_rng(3).choice(b.n, 5000, replace=False)
    marked, _ = dq.cancel(b.task_ids[gone])
    assert marked == 5000
    keep = np.setdiff1d(np.arange(b.n), gone)
    r = dq.drain("identity", b.n, endpoint=True)
    assert r.n_popped == b.n and r.n == keep.size and np.array_equal(r.task_ids, b.task_ids[keep])
    assert outcomes(r) == [full[i] for i in keep]
    assert dq.depth() == 0


def test_peek_async_bursts_mixed_with_task_queue_drains(dq):
    b = synth.strings_batch(20_000, 128, adversarial_frac=0.05, seed=8)
    dq.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, L.TF_HTTP_BODY, np.uint8))
    want_ep = outcomes(peek(dq, "identity", b.n, True))
    tq = peek(dq, "identity", b.n, False)
    want_tq = (tq.status.copy(), tq.fifo_payload().copy())
    assert dq.depth() == b.n
    for k in range(6):                                        # async bursts of k + 2 launches, endpoint / task-queue alternating
        for j in range(k + 2):
            dq.drain_launch("identity", b.n, peek=True, wait=False, endpoint=j % 2 == 0)
        r = dq.fetch()
        if (k + 1) % 2 == 0:                                  # the burst's last launch was an endpoint drain
            assert outcomes(r) == want_ep
        else:
            assert np.array_equal(r.status, want_tq[0]) and np.array_equal(r.fifo_payload(), want_tq[1])
    # a task-queue drain right after an endpoint drain equals one on a fresh ctx
    dq.drain_launch("identity", b.n, peek=True, endpoint=True)
    r = dq.drain("identity", b.n)
    from beta9_b200.device_queue import DeviceQueue
    with DeviceQueue(ring_bytes=1 << 28, ring_tasks=1 << 16, max_drain_tasks=1 << 16, max_result_bytes=1 << 27) as fresh:
        fresh.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, L.TF_HTTP_BODY, np.uint8))
        f = fresh.drain("identity", b.n)
    assert np.array_equal(r.status, f.status) and np.array_equal(r.has_result, f.has_result)
    assert np.array_equal(r.fifo_payload(), f.fifo_payload()) and dq.depth() == 0


def test_flags_are_checked(dq):
    lib = L.load()
    assert lib.b9_endpoint_drain_launch(dq._ctx, 0, 10, L.DRAIN_PICKLE_FULL) == L.B9_EINVAL
    assert lib.b9_endpoint_drain_launch(dq._ctx, 0, 10, 8) == L.B9_EINVAL
    assert lib.b9_endpoint_drain_launch(dq._ctx, 9, 10, 0) == L.B9_ENOSYS
    with pytest.raises(ValueError):
        dq.drain("identity", endpoint=True, full_pickle=True)


def test_non_http_tasks_are_unsupported(dq):
    b = synth.strings_batch(100, 32, seed=2)
    for flags in (0, L.TF_PICKLE, L.TF_TASK_MSG, L.TF_HTTP_BODY | L.TF_PICKLE):
        dq.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, flags, np.uint8))
        r = dq.drain("identity", b.n, endpoint=True)
        assert r.n == b.n and (r.status == L.ST_UNSUPPORTED).all() and not r.has_result.any()


def test_overflow_then_larger_fetch():
    from beta9_b200.device_queue import DeviceQueue
    b = synth.strings_batch(4000, 200, seed=4)
    with DeviceQueue(ring_bytes=1 << 24, ring_tasks=1 << 14, max_drain_tasks=1 << 14, max_result_bytes=1 << 16) as q:
        q.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, L.TF_HTTP_BODY, np.uint8))
        with pytest.raises(L.B9Error) as e:                    # staging too small: nothing consumed
            q.drain("identity", b.n, endpoint=True)
        assert e.value.code == L.B9_ENOSPC and q.depth() == b.n
        r = q.drain("identity", 200, endpoint=True)            # a window that fits
        assert r.n == 200 and q.depth() == b.n - 200
    with DeviceQueue(ring_bytes=1 << 24, ring_tasks=1 << 14, max_drain_tasks=1 << 14, max_result_bytes=1 << 22) as q:
        q.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, L.TF_HTTP_BODY, np.uint8))
        n = q.drain_launch("identity", b.n, endpoint=True)
        with pytest.raises(L.B9Error) as e:                    # the caller's buffers are too small: records stay
            q._fetch(n, 1024)
        assert e.value.code == L.B9_ENOSPC and q.depth() == b.n
        r = q._fetch(n, None)
        assert r.n == b.n and q.depth() == 0
        assert [o for o in outcomes(r)] == [quick_oracle(x, "identity") for x in b.tasks()]


def test_small_wrapping_ring():
    from beta9_b200.device_queue import DeviceQueue
    with DeviceQueue(ring_bytes=1 << 16, ring_tasks=256, max_drain_tasks=256, max_result_bytes=1 << 20) as q:
        for rnd in range(12):
            b = synth.strings_batch(150, 80 + 7 * rnd, adversarial_frac=0.1, seed=100 + rnd)
            q.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, L.TF_HTTP_BODY, np.uint8))
            r = q.drain("identity", 100, endpoint=True)
            r2 = q.drain("identity", 100, endpoint=True)
            assert r.n + r2.n == b.n and q.depth() == 0
            assert outcomes(r) + outcomes(r2) == [quick_oracle(x, "identity") for x in b.tasks()]


def test_drain_fetch_object(dq):
    b = synth.strings_batch(3000, 64, adversarial_frac=0.1, seed=9)
    bodies = b.tasks() + [b'{"args": [""]}', b'{"args": []}', b"{"]
    tid = push_bodies(dq, bodies)
    obj = dq.drain_object("identity", len(bodies), endpoint=True)
    lib = L.load()
    for i, body in enumerate(bodies):
        rec = L.SinkRecord()
        assert lib.b9_sink_get(obj.ctypes.data, obj.size, i, C.byref(rec)) == 0
        assert C.string_at(rec.task_id, 16) == tid[i].tobytes()
        want = quick_oracle(body, "identity")
        if want[0] == EP.OK:
            assert rec.status == L.ST_COMPLETE and rec.has_result == 1 and C.string_at(rec.data, rec.length) == want[1]
        else:
            assert rec.has_result == 0


def test_submit_from_threads_then_endpoint_requests(dq):
    from beta9_b200.endpoint import Endpoint
    bodies = [json.dumps({"args": [f"t{k}-{i}-é"]}, ensure_ascii=(i % 2 == 0)).encode() for k in range(4) for i in range(500)]
    ids = [uuid.uuid4().bytes for _ in bodies]

    def worker(k):
        for i in range(k, len(bodies), 4):
            dq.submit(ids[i], bodies[i], L.TF_HTTP_BODY)
    th = [threading.Thread(target=worker, args=(k,)) for k in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    dq.flush()
    r = dq.drain("identity", len(bodies), endpoint=True)
    got = {r.task_ids[i].tobytes(): o for i, o in enumerate(outcomes(r))}
    assert len(got) == len(bodies)
    for tid, body in zip(ids, bodies):
        assert got[tid] == (EP.OK, json.dumps(json.loads(body)["args"][0], ensure_ascii=False).encode())
    ep = Endpoint(gpu_handler="json_sum", queue=dq)(lambda x: x)
    reqs = [b'{"args": [{"values": [1, 2.5]}]}', b'{"args": [{"values": []}]}', b"not json", b'{"args": [1]}',
            b'{"args": [{"values": [1e308, 1e308]}]}']
    assert ep.requests(reqs) == [(200, b"3.5"), (200, b"0"), (400, b'{"error":"invalid request payload"}'), (500, None), (None, None)]
    assert ep.unsupported == [reqs[-1]]
    assert Endpoint(gpu_handler="identity", queue=dq)(lambda x: x).request(b'{"args": ["\\u00e9"]}') == (200, '"é"'.encode())
