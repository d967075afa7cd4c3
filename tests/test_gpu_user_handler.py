"""GPU tests of user handlers (b9_handler_load, include/b9gpu_handler.cuh): the example handlers (examples/handlers), loaded
from the cubin build() makes, drained on the device and compared with their Python twins through the oracle's loops (the
same comparisons tests/test_user_handler_on_host.py makes on a CPU), plus the drain contract they share with the built-in
handlers: mixed windows, cancelled slots, peek and async bursts beside built-in drains, a wrapping ring, B9_ENOSPC, the
retry policy, callbacks, the endpoint drain, BASELINE-size batches against the built-in drains, and the loader's errors."""
import base64
import hashlib
import hmac
import json
import os

import numpy as np
import pytest

from beta9_b200 import _lib as L
from beta9_b200 import build as B
from beta9_b200 import synth
from oracle.pyoracle import callback as CB
from oracle.pyoracle.gojson import go_unmarshal_task_payload
from tests import test_user_handler_on_host as H

pytestmark = pytest.mark.gpu
NAMES = H.NAMES
KEY = b"workspace-signing-key"


def new_queue(**kw):
    from beta9_b200.device_queue import DeviceQueue
    q = DeviceQueue(**kw)
    for name in NAMES:
        q.load_handler(B.EXAMPLE_CUBIN, name)
    return q


@pytest.fixture(scope="module")
def dq():
    q = new_queue(ring_bytes=1 << 31, ring_tasks=1 << 22, max_drain_tasks=1 << 21, max_result_bytes=1 << 30)
    yield q
    q.close()


def records(r):
    return [(int(r.status[i]), int(r.has_result[i]), None, r.result(i) or b"") for i in range(r.n)]


def push(q, payloads, flags=0, ids=None):
    b = synth.from_payloads(list(payloads))
    tid = b.task_ids if ids is None else np.frombuffer(b"".join(ids), np.uint8).reshape(-1, 16)
    q.push_batch(tid, b.payload, b.offsets, flags=np.full(b.n, flags, np.uint8))
    return tid


def device(q):
    """the host shim's signature (tests/test_user_handler_on_host.py), answered by one device drain"""
    def run(payloads, name, rendering, flags=0, ids=None):
        if not payloads:
            return []
        assert q.depth() == 0
        push(q, payloads, flags, ids)
        r = q.drain(name, endpoint=rendering == H.ENDPOINT)
        assert r.n == len(payloads) and q.depth() == 0
        return records(r)
    return run


@pytest.mark.parametrize("name", NAMES)
def test_payloads_bodies_records_and_endpoint(dq, name):
    uh = device(dq)
    c = H.corpus()
    assert H.check_tq(uh, name, c) > len(c) * 9 // 10
    assert H.check_tq(uh, name, c, http=True) > len(c) * 8 // 10
    assert H.check_ep(uh, name, c) > len(c) * 8 // 10
    recs, ids = H.records_of(c)
    assert H.check_records(uh, name, recs, ids) > len(recs) * 9 // 10


def test_f64_corpus_and_mutations(dq):
    from tests.f64_corpus import _literals
    uh = device(dq)
    rng = np.random.default_rng(11)
    lits = _literals()
    pick = [lits[i] for i in rng.choice(len(lits), 20000, replace=False)]
    bodies = [b'{"args": [[%s, 3, 0.5]]}' % s.encode() for s in pick] + [b'{"args": [%s]}' % s.encode() for s in pick[:4000]]
    for name in NAMES:
        H.check_tq(uh, name, bodies)
        H.check_ep(uh, name, bodies)
    base = [b for b in H.corpus() if len(b) >= 4][:400]
    muts = []
    for _ in range(20000):
        m = bytearray(base[int(rng.integers(0, len(base)))])
        pos = int(rng.integers(0, len(m)))
        m[pos] = int(rng.choice(list(b'{}[],:" 01e.-\\') + [0xC3, 0xFF]))
        muts.append(bytes(m))
    for name in NAMES:
        H.check_tq(uh, name, muts)


def _mixed():
    c = H.corpus()[:600]
    recs, ids = H.records_of(c[:300])
    return c, recs, ids


@pytest.mark.parametrize("name", NAMES)
def test_mixed_window_and_pickle_tasks(dq, name):
    """one window of SDK payloads, HTTP bodies, records and pickle tasks: each task's record is what a window of its own
    kind gives, and every pickle task is UNSUPPORTED"""
    c, recs, ids = _mixed()
    uh = device(dq)
    want = uh(c, name, H.TQ) + uh(c, name, H.TQ, H.TF_HTTP_BODY) + uh(recs, name, H.TQ, H.TF_TASK_MSG, ids) + \
        [(H.UNSUPPORTED, 0, None, b"")] * 50
    kinds = [(p, 0, None) for p in c] + [(p, H.TF_HTTP_BODY, None) for p in c] + [(r, H.TF_TASK_MSG, i) for r, i in zip(recs, ids)] + \
        [(b"\x80\x05\x95" + bytes(20), 0x04, None)] * 50
    order = np.random.default_rng(5).permutation(len(kinds))
    for k in order:                                                       # one push per task, in the shuffled order
        p, fl, tid = kinds[k]
        push(dq, [p], fl, [tid] if tid else [int(k + 7).to_bytes(16, "big")])
    r = dq.drain(name)
    assert r.n == len(kinds)
    assert records(r) == [want[k] for k in order]


@pytest.mark.parametrize("name", NAMES)
def test_cancelled_slots_count_mode(dq, name):
    c = H.corpus()[:2000]
    full = device(dq)(c, name, H.TQ)
    ids = push(dq, c)
    keep = np.ones(len(c), bool)
    keep[np.random.default_rng(2).choice(len(c), 333, replace=False)] = False
    dq.cancel(ids[~keep])
    r = dq.drain(name)
    assert r.n == int(keep.sum()) and r.n_popped == len(c)
    assert records(r) == [full[i] for i in np.flatnonzero(keep)]
    assert np.array_equal(r.task_ids, ids[keep])


def test_peek_and_async_bursts_beside_built_in_drains(dq):
    c = [p for p in H.corpus() if p.startswith(b'{"args": ["')][:3000]
    uh = device(dq)
    want = {n: uh(c, n, H.TQ) for n in NAMES}
    ep_want = uh(c, "echo_str", H.ENDPOINT, H.TF_HTTP_BODY)
    push(dq, c)
    ident = device_builtin(dq, "identity")
    for rnd in range(3):
        for n in NAMES:
            dq.drain_launch(n, peek=True)
            assert records(dq.fetch()) == want[n]
            assert records(device_builtin(dq, "identity")) == records(ident)
        for n in NAMES + ["crc32"]:                                           # an async burst: the last launch's records wait
            dq.drain_launch(n, peek=True, wait=False)
        assert records(dq.fetch()) == records(device_builtin(dq, "crc32"))
        dq.drain_launch(NAMES[rnd], peek=True, wait=False)
        dq.drain_launch("identity", peek=True, wait=False)
        dq.drain_launch(NAMES[rnd], peek=True, wait=False)
        assert records(dq.fetch()) == want[NAMES[rnd]]
    assert dq.depth() == len(c)
    dq.drain("identity")
    push(dq, c, H.TF_HTTP_BODY)
    dq.drain_launch("echo_str", peek=True, endpoint=True, wait=False)
    dq.drain_launch("echo_str", peek=True, endpoint=True, wait=False)
    assert records(dq.fetch()) == ep_want
    dq.drain("echo_str", endpoint=True)
    assert dq.depth() == 0


def device_builtin(q, handler):
    q.drain_launch(handler, peek=True)
    return q.fetch()


def test_wrapping_ring():
    """a 4 KiB, 32-slot ring: each step pushes a part and drains the part pushed before it, so that windows wrap both the
    slots and the bytes; every record against the twin"""
    from oracle.pyoracle.loop import run_task_loop
    q = new_queue(ring_bytes=4096, ring_tasks=32, max_drain_tasks=32, max_result_bytes=1 << 16)
    try:
        c = [p for p in H.corpus() if len(p) < 200][:600]
        rng = np.random.default_rng(9)
        pending, i, steps = [], 0, 0
        while i < len(c) or pending:
            if i < len(c):
                k = int(rng.integers(1, 7))
                part = c[i:i + k]
                i += k
                push(q, part)
                pending.append(part)
            if len(pending) > 1 or i >= len(c):
                part = pending.pop(0)
                name = NAMES[int(rng.integers(0, 4))]
                r = q.drain(name, max_tasks=len(part))
                assert r.n == len(part)
                want = run_task_loop(part, [bytes(16)] * len(part), handler=H.twins.TWINS[name])
                for p, w, g in zip(part, want, records(r)):
                    if g[0] == H.UNSUPPORTED:
                        assert H.may_decline(name, p, None) or name == "prod", (name, p)
                        continue
                    assert (g[0], g[3] or None) == ({"COMPLETE": 0, "ERROR": 1, "REJECTED": 3}[w.status], w.result), (name, p)
                steps += 1
        assert q.depth() == 0 and steps > 100
    finally:
        q.close()


def test_enospc_consumes_nothing(dq):
    c = [H.sdk("x" * 300)] * 100
    push(dq, c)
    dq.drain_launch("echo_str")
    assert dq.running() == 100
    with pytest.raises(L.B9Error) as e:
        dq.fetch(cap_bytes=1000)
    assert e.value.code == L.B9_ENOSPC and dq.depth() == 100
    r = dq.fetch()
    assert r.n == 100 and dq.depth() == 0 and r.result(0) == json.dumps("x" * 300).encode()
    # the staging itself too small: the launch reports it and nothing is consumed
    q = new_queue(ring_bytes=1 << 20, ring_tasks=1024, max_drain_tasks=1024, max_result_bytes=4096)
    try:
        push(q, c)
        with pytest.raises(L.B9Error) as e:
            q.drain_launch("echo_str")
        assert e.value.code == L.B9_ENOSPC and q.depth() == 100
        r = q.drain("echo_str", max_tasks=10)
        assert r.n == 10 and q.depth() == 90
    finally:
        q.close()


def test_retry_policy_on_a_user_handlers_class(dq):
    """word_count raises AttributeError for a non-str: under retry_for=[AttributeError] those tasks come back RETRY, are
    pushed again, and end RETRY_LIMIT; the str tasks complete"""
    dq.set_retry_policy([AttributeError], 2)
    try:
        c = [H.sdk("a b"), H.sdk(7), H.sdk([1]), H.sdk("c")]
        ids = push(dq, c)
        seen = []
        for _ in range(4):
            r = dq.drain("word_count")
            seen.append([(r.task_ids[i].tobytes(), int(r.status[i])) for i in range(r.n)])
            if dq.depth() == 0:
                break
        assert seen[0] == [(ids[0].tobytes(), 0), (ids[1].tobytes(), L.ST_RETRY), (ids[2].tobytes(), L.ST_RETRY), (ids[3].tobytes(), 0)]
        assert seen[1] == [(ids[1].tobytes(), L.ST_RETRY), (ids[2].tobytes(), L.ST_RETRY)]
        assert seen[2] == [(ids[1].tobytes(), L.ST_RETRY_LIMIT), (ids[2].tobytes(), L.ST_RETRY_LIMIT)]
        assert dq.depth() == 0
        # a class the policy does not name stays ERROR: echo_str raises TypeError
        push(dq, [H.sdk(7)])
        assert int(dq.drain("echo_str").status[0]) == L.ST_ERROR
    finally:
        dq.set_retry_policy([], 0)


def test_callbacks_task_queue_and_endpoint(dq):
    c = H.corpus()[:800] + [H.sdk([1e308, 10.0]), H.sdk([2, 0.5])]
    dq.set_callback_policy(KEY)
    try:
        for name in NAMES:
            ids = push(dq, c)
            r = dq.drain(name, callbacks=True)
            assert r.n == len(c) and r.cb_timestamp > 0
            for i in range(r.n):
                st = {0: "COMPLETE", 1: "ERROR", 3: "REJECTED", 4: "UNSUPPORTED"}[int(r.status[i])]
                kw = go_unmarshal_task_payload(c[i])[1] if st == "ERROR" else None      # (the kwargs Go decoded)
                assert int(r.cb_kind[i]) == CB.callback_kind(st, r.result(i), kw), (name, c[i])
                if int(r.cb_kind[i]) == L.CB_POST:
                    sig, _ = CB.sign_payload(CB.callback_body(r.result(i)), KEY, r.cb_timestamp)
                    assert r.cb_digest[i].tobytes().hex() == sig
            assert np.array_equal(r.task_ids, ids)
        # the endpoint runner's callbacks: D = json.dumps of the response value, signed as {"data": D}
        for runners in (False, True):
            dq.set_callback_runners(endpoint=runners)
            for name in NAMES:
                push(dq, c, H.TF_HTTP_BODY)
                if not runners:
                    r = dq.drain(name, endpoint=True)
                    assert r.cb_kind is None
                    continue
                r = dq.drain(name, endpoint=True, callbacks=True)
                for i in range(r.n):
                    st = int(r.status[i])
                    want = L.CB_POST if st == 0 else L.CB_NONE if st == L.ST_REJECTED else L.CB_HOST
                    assert int(r.cb_kind[i]) == want
                    if want == L.CB_POST:
                        d = json.dumps(json.loads(r.result(i))).encode()
                        body = r.callback_body(i)
                        assert body == b'{"data": ' + d + b"}"
                        msg = base64.b64encode(body) + b":%d" % r.cb_timestamp
                        assert r.cb_digest[i].tobytes() == hmac.new(KEY, msg, hashlib.sha256).digest()
        dq.set_callback_runners()
    finally:
        dq.set_callback_policy(None)


def test_baseline_size_against_built_in_drains(dq):
    """configs[2]'s 1 M zipf strings: crc32_str == crc32; configs[1]'s 1 M strings: echo_str == identity, record for record"""
    for batch, mine, builtin in ((synth.crc_batch(1 << 20), "crc32_str", "crc32"),
                                 (synth.strings_batch(1 << 20, 256), "echo_str", "identity")):
        dq.push_batch(batch.task_ids, batch.payload, batch.offsets)
        a = device_builtin(dq, builtin)
        b = device_builtin(dq, mine)
        assert a.n == b.n == batch.n
        assert np.array_equal(a.status, b.status) and np.array_equal(a.has_result, b.has_result)
        assert np.array_equal(a.lengths, b.lengths) and np.array_equal(a.fifo_payload(), b.fifo_payload())
        assert np.array_equal(a.task_ids, b.task_ids)
        dq.drain(builtin)
        assert dq.depth() == 0


def test_loader_errors_and_ids():
    from beta9_b200.device_queue import DeviceQueue
    image = open(B.EXAMPLE_CUBIN, "rb").read()
    with DeviceQueue(ring_bytes=1 << 22, ring_tasks=1 << 12, max_drain_tasks=1 << 12, max_result_bytes=1 << 22) as a, \
            DeviceQueue(ring_bytes=1 << 22, ring_tasks=1 << 12, max_drain_tasks=1 << 12, max_result_bytes=1 << 22) as b:
        c = [H.sdk(s) for s in ["x", "ab c", "", "é"]] + [H.sdk(1), H.sdk([1, 2])]
        push(a, c)
        before = [records(device_builtin(a, h)) for h in ("identity", "crc32")]
        for bad, what in ((bytes(np.random.default_rng(1).integers(0, 256, 4096, dtype=np.uint8)), "not an ELF"),
                          (image[:len(image) // 2], "not an ELF"),
                          (image.replace(b"b9h_v%d_" % B.handler_abi_version(), b"b9h_v%d_" % (B.handler_abi_version() + 8)), "version")):
            with pytest.raises(L.B9Error) as e:
                a.load_handler(bad, "echo_str")
            assert e.value.code == L.B9_EINVAL and what in str(e.value), str(e.value)
        with pytest.raises(L.B9Error) as e:
            a.load_handler(image, "no_such_handler")
        assert e.value.code == L.B9_EINVAL and "no_such_handler" in str(e.value)
        with pytest.raises(L.B9Error) as e:
            a.load_handler(image, "bad-name")
        assert e.value.code == L.B9_EINVAL
        hid = a.load_handler(image, "word_count")
        assert hid == L.H_USER_BASE
        assert a.load_handler(image, "prod") == L.H_USER_BASE + 1
        assert [records(device_builtin(a, h)) for h in ("identity", "crc32")] == before
        assert a._lib.b9_handler_name(hid) is None and a._lib.b9_handler_id(b"word_count") == L.B9_ENOSYS
        # an id of another context, one never returned, and the pickle pass
        push(b, c)
        for q, h in ((b, hid), (a, L.H_USER_BASE + 2), (a, 4), (a, 255)):
            with pytest.raises(L.B9Error) as e:
                q.drain_launch(h)
            assert e.value.code == L.B9_ENOSYS
        with pytest.raises(L.B9Error) as e:
            a.drain_launch(hid, full_pickle=True)
        assert e.value.code == L.B9_EINVAL and a.depth() == len(c) and a.running() == 0
        r = a.drain(hid)
        assert [int(x) for x in r.status] == [0, 0, 0, 0, 1, 1] and r.result(1) == b"2"


def test_sdk_mirrors():
    from beta9_b200.endpoint import Endpoint
    from beta9_b200.taskqueue import TaskQueue
    tq = TaskQueue(gpu_handler="word_count", gpu_handler_image=B.EXAMPLE_CUBIN)
    f = tq(H.twins.word_count)
    f.put("a b c")
    f.put("")
    f.put(3)
    got = f.process_tasks()
    assert [(t.status, t.result) for t in got] == [("COMPLETE", 3), ("COMPLETE", None), ("ERROR", None)], got
    os.environ["B9_GPU_HANDLER"], os.environ["B9_GPU_HANDLER_IMAGE"] = "echo_str", B.EXAMPLE_CUBIN
    try:
        ep = Endpoint()(H.twins.echo_str)
    finally:
        del os.environ["B9_GPU_HANDLER"], os.environ["B9_GPU_HANDLER_IMAGE"]
    assert ep.requests([b'{"args": ["caf\\u00e9"]}', b'{"args": [1]}', b"{"]) == [(200, '"café"'.encode()), (500, None),
                                                                                   (400, b'{"error":"invalid request payload"}')]
