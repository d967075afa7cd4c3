"""GPU tests of user handlers with a declared signature (B9H_SIGNATURE, include/b9gpu_handler.cuh): greet, join and
field_sum from the example image build() makes, drained on the device and compared with their Python twins through the
oracle's loops (the comparisons tests/test_user_signature_on_host.py makes on a CPU), plus the drain contract: mixed
windows and cancelled slots in count mode, PEEK / ASYNC beside built-in and one-Arg user drains, a small wrapping ring,
B9_ENOSPC, the retry policy on binding failures, callbacks, and the SDK mirrors."""
import json

import numpy as np
import pytest

from beta9_b200 import _lib as L
from beta9_b200 import build as B
from oracle.pyoracle import callback as CB
from oracle.pyoracle.gojson import go_unmarshal_task_payload
from tests import test_gpu_user_handler as G
from tests import test_user_handler_on_host as U
from tests import test_user_signature_on_host as S

pytestmark = pytest.mark.gpu
NAMES = ["greet", "join", "field_sum"]
KEY = b"workspace-signing-key"


def new_queue(**kw):
    from beta9_b200.device_queue import DeviceQueue
    q = DeviceQueue(**kw)
    for name in NAMES + U.NAMES:
        q.load_handler(B.EXAMPLE_CUBIN, name)
    return q


@pytest.fixture(scope="module")
def dq():
    q = new_queue(ring_bytes=1 << 30, ring_tasks=1 << 20, max_drain_tasks=1 << 20, max_result_bytes=1 << 29)
    yield q
    q.close()


def device(q):
    run = G.device(q)
    return lambda payloads, name, rendering, flags=0, ids=None: run(payloads, name, rendering, flags, ids)


@pytest.mark.parametrize("name", NAMES)
def test_payloads_bodies_records_and_endpoint(dq, name):
    S.check_all(device(dq), name, S.corpus(), min_share=0.9)


def test_binding_failures_and_mutations(dq):
    us = device(dq)
    cases = {"greet": [S.call("a", "b", "c"), S.call(), S.call("a", bogus=1), S.call("a", name="b")],
             "join": [S.call(sep="-", parts=["a"])], "field_sum": [S.call([{"x": 1}], "x"), S.call([{"x": 1}])]}
    for name, calls in cases.items():
        for args, kwargs in calls:
            bodies = S.renderings(args, kwargs)
            assert all(g[0] == U.ERROR for g in us(bodies[:2], name, U.TQ))
            assert all(g[0] == U.ERROR for g in us(bodies, name, U.TQ, U.TF_HTTP_BODY))
            assert all(g[0] == U.ERROR for g in us(bodies, name, U.ENDPOINT, U.TF_HTTP_BODY))
    rng = np.random.default_rng(17)
    base = [b for b in S.corpus() if len(b) >= 4]
    muts = []
    for _ in range(12000):
        m = bytearray(base[int(rng.integers(0, len(base)))])
        m[int(rng.integers(0, len(m)))] = int(rng.choice(list(b'{}[],:" 01e.-\\xdn') + [0xC3, 0xFF]))
        muts.append(bytes(m))
    for name in NAMES:
        S.check_tq(us, name, muts)
        S.check_tq(us, name, muts, http=True)
        S.check_ep(us, name, muts)


def test_hypothesis_like_random_calls(dq):
    """seeded random (args, kwargs) calls over the parameter names and value shapes the host test draws from"""
    rng = np.random.default_rng(23)
    keys = ["name", "greeting", "punct", "sep", "parts", "rows", "field", "x", "args", "kwargs", "context", "", "é"]
    vals = ["a", "", "é", 1, 2.5, None, True, [{"x": 1}, {"x": 2.5}], [{"y": 1}], ["p", "q"], {"x": 3}, 2**63]
    bodies = []
    for _ in range(3000):
        args = [vals[int(i)] for i in rng.integers(0, len(vals), int(rng.integers(0, 4)))]
        kwargs = {keys[int(i)]: vals[int(j)] for i, j in zip(rng.integers(0, len(keys), 3), rng.integers(0, len(vals), 3))
                  if rng.random() < 0.6}
        bodies += S.renderings(args, kwargs)
    for name in NAMES:
        S.check_all(device(dq), name, bodies)


@pytest.mark.parametrize("name", NAMES)
def test_mixed_window_and_cancelled_slots_count_mode(dq, name):
    """one window of SDK payloads, HTTP bodies and records, one push per task in a shuffled order, a third of it
    cancelled: each record is what a window of its own kind gives"""
    c = S.corpus()
    recs, ids = U.records_of(c)
    us = device(dq)
    want = us(c, name, U.TQ) + us(c, name, U.TQ, U.TF_HTTP_BODY) + us(recs, name, U.TQ, U.TF_TASK_MSG, ids)
    kinds = [(p, 0, None) for p in c] + [(p, U.TF_HTTP_BODY, None) for p in c] + [(r, U.TF_TASK_MSG, i) for r, i in zip(recs, ids)]
    order = np.random.default_rng(5).permutation(len(kinds))
    tids = []
    for k in order:
        p, fl, tid = kinds[k]
        tids.append(G.push(dq, [p], fl, [tid] if tid else [((1 << 64) + int(k)).to_bytes(16, "big")])[0])   # (ids no record carries)
    tids = np.stack(tids)
    keep = np.ones(len(kinds), bool)
    keep[np.random.default_rng(2).choice(len(kinds), len(kinds) // 3, replace=False)] = False
    dq.cancel(tids[~keep])
    r = dq.drain(name)
    assert r.n == int(keep.sum()) and r.n_popped == len(kinds)
    assert G.records(r) == [want[order[i]] for i in np.flatnonzero(keep)]


def test_peek_and_async_beside_built_in_and_one_arg_drains(dq):
    c = [S.sdk(["n%d" % i], {"punct": "?"}) for i in range(500)] + [S.sdk(["x"], {}), S.sdk([], {"name": "y"})]
    us = device(dq)
    want = {n: us(c, n, U.TQ) for n in NAMES + ["echo_str"]}
    G.push(dq, c)
    ident = G.device_builtin(dq, "identity")
    for rnd in range(3):
        for n in NAMES + ["echo_str"]:
            dq.drain_launch(n, peek=True)
            assert G.records(dq.fetch()) == want[n]
        for n in NAMES + ["echo_str", "identity"]:
            dq.drain_launch(n, peek=True, wait=False)
        assert G.records(dq.fetch()) == G.records(ident)
        dq.drain_launch("echo_str", peek=True, wait=False)
        dq.drain_launch(NAMES[rnd], peek=True, wait=False)
        assert G.records(dq.fetch()) == want[NAMES[rnd]]
    assert dq.depth() == len(c)
    r = dq.drain("greet")
    assert G.records(r) == want["greet"] and dq.depth() == 0
    assert r.result(0) == b'"Hello, n0?"'


def test_wrapping_ring():
    from oracle.pyoracle.loop import run_task_loop
    q = new_queue(ring_bytes=4096, ring_tasks=32, max_drain_tasks=32, max_result_bytes=1 << 16)
    try:
        c = [p for p in S.corpus() if len(p) < 200]
        rng = np.random.default_rng(9)
        pending, i, steps = [], 0, 0
        while i < len(c) or pending:
            if i < len(c):
                k = int(rng.integers(1, 7))
                part = c[i:i + k]
                i += k
                G.push(q, part)
                pending.append(part)
            if len(pending) > 1 or i >= len(c):
                part = pending.pop(0)
                name = NAMES[int(rng.integers(0, 3))]
                r = q.drain(name, max_tasks=len(part))
                assert r.n == len(part)
                want = run_task_loop(part, [bytes(16)] * len(part), handler=S.FNS[name], keep_wire=True)
                for p, w, g in zip(part, want, G.records(r)):
                    if g[0] == U.UNSUPPORTED:
                        t = json.loads(w.wire) if w.wire else None
                        assert S.may_decline(name, p, t and (t["args"] or []), t and (t["kwargs"] or {}), sdk=True), (name, p)
                        continue
                    assert (g[0], g[3] or None) == ({"COMPLETE": 0, "ERROR": 1, "REJECTED": 3}[w.status], w.result), (name, p)
                steps += 1
        assert q.depth() == 0 and steps > 50
    finally:
        q.close()


def test_enospc_consumes_nothing(dq):
    c = [S.sdk([], {"name": "x" * 300})] * 100
    G.push(dq, c)
    dq.drain_launch("greet")
    with pytest.raises(L.B9Error) as e:
        dq.fetch(cap_bytes=1000)
    assert e.value.code == L.B9_ENOSPC and dq.depth() == 100
    r = dq.fetch()
    assert r.n == 100 and dq.depth() == 0 and r.result(0) == json.dumps("Hello, " + "x" * 300 + "!").encode()


def test_retry_policy_on_binding_failures(dq):
    """a binding failure is a TypeError: under retry_for=[TypeError] it comes back RETRY, is pushed again, and ends
    RETRY_LIMIT; calls that bind complete"""
    dq.set_retry_policy([TypeError], 2)
    try:
        c = [S.sdk(["a"], {}), S.sdk(["a", "b", "c"], {}), S.sdk([], {"punct": "?"}), S.sdk(["b"], {"punct": "?"})]
        ids = G.push(dq, c)
        seen = []
        for _ in range(4):
            r = dq.drain("greet")
            seen.append([(r.task_ids[i].tobytes(), int(r.status[i])) for i in range(r.n)])
            if dq.depth() == 0:
                break
        assert seen[0] == [(ids[0].tobytes(), 0), (ids[1].tobytes(), L.ST_RETRY), (ids[2].tobytes(), L.ST_RETRY), (ids[3].tobytes(), 0)]
        assert seen[1] == [(ids[1].tobytes(), L.ST_RETRY), (ids[2].tobytes(), L.ST_RETRY)]
        assert seen[2] == [(ids[1].tobytes(), L.ST_RETRY_LIMIT), (ids[2].tobytes(), L.ST_RETRY_LIMIT)]
        assert dq.depth() == 0
        dq.set_retry_policy([KeyError], 2)                       # a class the policy does not name stays ERROR
        G.push(dq, [S.sdk(["a", "b", "c"], {})])
        assert int(dq.drain("greet").status[0]) == L.ST_ERROR
    finally:
        dq.set_retry_policy([], 0)


def test_callbacks(dq):
    c = S.corpus()[:300] + [S.sdk(["a"], {"callback_url": "http://x"})]
    dq.set_callback_policy(KEY)
    try:
        for name in NAMES:
            ids = G.push(dq, c)
            r = dq.drain(name, callbacks=True)
            assert r.n == len(c) and r.cb_timestamp > 0
            for i in range(r.n):
                st = {0: "COMPLETE", 1: "ERROR", 3: "REJECTED", 4: "UNSUPPORTED"}[int(r.status[i])]
                kw = go_unmarshal_task_payload(c[i])[1] if st == "ERROR" else None
                assert int(r.cb_kind[i]) == CB.callback_kind(st, r.result(i), kw), (name, c[i])
                if int(r.cb_kind[i]) == L.CB_POST:
                    sig, _ = CB.sign_payload(CB.callback_body(r.result(i)), KEY, r.cb_timestamp)
                    assert r.cb_digest[i].tobytes().hex() == sig
            assert np.array_equal(r.task_ids, ids)
    finally:
        dq.set_callback_policy(None)


def test_sdk_mirrors():
    from beta9_b200.endpoint import Endpoint
    from beta9_b200.taskqueue import TaskQueue
    tq = TaskQueue(gpu_handler="greet", gpu_handler_image=B.EXAMPLE_CUBIN)
    f = tq(U.twins.greet)
    f.put(name="Ada", punct="?")
    f.put("Bo", "Hi")
    f.put("Cy", bogus=1)
    f.put(name=3)
    got = f.process_tasks()
    assert [(t.status, t.result) for t in got] == [("COMPLETE", "Hello, Ada?"), ("COMPLETE", "Hi, Bo!"), ("ERROR", None),
                                                   ("ERROR", None)], got
    ep = Endpoint(gpu_handler="greet", gpu_handler_image=B.EXAMPLE_CUBIN)(U.twins.greet)
    assert ep.request(b'{"name": "caf\\u00e9", "greeting": "Hej"}') == (200, '"Hej, café!"'.encode())
    assert ep.requests([b'{"name": "x", "extra": 1}', b'{"args": ["y"], "kwargs": {"punct": "."}}', b"{"]) == \
        [(500, None), (200, b'"Hello, y."'), (400, b'{"error":"invalid request payload"}')]
