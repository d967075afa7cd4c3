"""Device TaskMessage.Encode (b9_wire_encode) against the oracle's queue wire bytes, bit for bit."""
import numpy as np
import pytest

from beta9_b200 import synth
from oracle import coracle
from oracle.pyoracle import loop
from oracle.pyoracle.wire import QueueEnv
from tests import golden_util as G

pytestmark = pytest.mark.gpu

NOW = coracle.DEFAULT_NOW_NS
TTL = 7200


@pytest.fixture(scope="module")
def dq():
    from beta9_b200.device_queue import DeviceQueue
    q = DeviceQueue(ring_bytes=1 << 30, ring_tasks=1 << 20, max_drain_tasks=1 << 20, max_result_bytes=2 << 30)
    yield q
    q.close()


def push_with_meta(dq, b):
    n = b.n
    dq.push_batch(b.task_ids, b.payload, b.offsets, timestamp_unix=np.full(n, NOW // 10**9, np.int64),
                  expires_unix_ns=np.full(n, NOW + TTL * 10**9, np.int64))


def check(dq, b, allow_unsupported=False):
    push_with_meta(dq, b)
    r = dq.wire_encode(coracle.DEFAULT_WS, coracle.DEFAULT_STUB, ttl=TTL)
    assert dq.depth() == b.n                       # a peek: nothing consumed
    dq.drain("identity")                            # clear the queue
    o = coracle.run_batch(b.task_ids, b.payload, b.offsets, "identity", keep_wire=True, nthreads=8)
    assert r.n == b.n and np.array_equal(r.task_ids, b.task_ids)
    n_unsup = 0
    for i in range(b.n):
        want = o.wire_msg(i)
        if r.status[i] == 4:
            assert allow_unsupported, b.task(i)
            n_unsup += 1
            continue
        if o.status[i] == 3:                        # the reference would never have created the task
            assert r.status[i] == 3 and r.result(i) is None, b.task(i)
        elif o.status[i] == 4:                      # the C oracle itself declines (floats): nothing to compare
            continue
        else:
            assert r.status[i] == 0 and r.result(i) == want, (b.task(i), r.result(i), want)
    return n_unsup


def test_wire_identity_strings(dq):
    check(dq, synth.strings_batch(20_000, 64, adversarial_frac=0.3))
    check(dq, synth.strings_batch(3000, 256, adversarial_frac=0.5, seed=9))


def test_wire_other_configs(dq):
    check(dq, synth.crc_batch(5000))
    check(dq, synth.vadd_batch(2000))
    # json docs: {"id": .., "values": [...], "pad": ".."} is not in sorted key order -> the device declines, never guesses
    n = check(dq, synth.json_batch(200), allow_unsupported=True)
    assert n == 200


def test_wire_handcrafted_and_golden(dq):
    from tests.test_oracle_c_vs_py import HANDCRAFTED
    check(dq, synth.from_payloads(HANDCRAFTED), allow_unsupported=True)
    g = G.load()
    for name, cases in g["groups"].items():
        b = G.group_batch(cases)
        push_with_meta(dq, b)
        r = dq.wire_encode(g["workspace"], g["stub"], ttl=TTL)
        dq.drain("identity")
        import base64
        for i, c in enumerate(cases):
            if r.status[i] == 4:
                continue
            want = base64.b64decode(c["wire"]) if c["wire"] else None
            assert r.result(i) == want, (name, i)


def test_wire_overflow_leaves_the_queue_alone():
    """Records that exceed max_result_bytes: B9_ENOSPC and nothing consumed; a window that fits is then encoded."""
    from beta9_b200.device_queue import DeviceQueue
    from beta9_b200._lib import B9_ENOSPC, B9Error
    b = synth.strings_batch(2000, 64, adversarial_frac=0.3, seed=13)
    o = coracle.run_batch(b.task_ids, b.payload, b.offsets, "identity", keep_wire=True, nthreads=8)
    with DeviceQueue(ring_bytes=1 << 24, ring_tasks=1 << 12, max_drain_tasks=1 << 12, max_result_bytes=1 << 16) as q:
        push_with_meta(q, b)
        with pytest.raises(B9Error) as e:
            q.wire_encode(coracle.DEFAULT_WS, coracle.DEFAULT_STUB, ttl=TTL)
        assert e.value.code == B9_ENOSPC and q.depth() == b.n
        r = q.wire_encode(coracle.DEFAULT_WS, coracle.DEFAULT_STUB, ttl=TTL, max_tasks=64)
        assert r.n == 64 and q.depth() == b.n and np.array_equal(r.task_ids, b.task_ids[:64])
        assert np.array_equal(r.status, o.status[:64]) and (r.status == 0).sum() > 32
        assert all(r.result(i) == o.wire_msg(i) for i in range(64) if r.status[i] == 0)


def test_wire_sorted_objects_and_kwargs(dq):
    payloads = [loop.sdk_put_payload({"a": 1, "b": [1, 2, {"x": "<", "y": None}], "c": True}, k="v"),
                loop.sdk_put_payload(a=1, b="é "), loop.sdk_put_payload([{"": 0, "a": -5}]),
                b'{"kwargs": {"b": 1, "a": 2}, "args": []}',          # unsorted keys: declined
                b'{"args": [1.5]}', b'{"args": null, "kwargs": null}', b"null", b"{}"]
    b = synth.from_payloads(payloads)
    push_with_meta(dq, b)
    r = dq.wire_encode(coracle.DEFAULT_WS, coracle.DEFAULT_STUB, ttl=TTL)
    dq.drain("identity")
    ids = [bytes(x) for x in b.task_ids]
    want = loop.run_task_loop(payloads, ids, "identity", keep_wire=True, now_unix_ns=NOW)
    for i in (0, 1, 2, 5, 6, 7):
        assert r.status[i] == 0 and r.result(i) == want[i].wire, (payloads[i], r.result(i), want[i].wire)
    assert r.status[3] == 4 and r.status[4] == 4
