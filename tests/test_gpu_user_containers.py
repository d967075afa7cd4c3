"""GPU tests of user handlers that return lists and dicts (the sinks' list / dict / value calls, include/b9gpu_handler.cuh):
the container script handler from tests/handlers/containers.cubin and the examples tokens, grid, describe and pick from
the example image, both made by build(). Every device record must equal the host shim's, which
tests/test_user_containers_on_host.py pins to the twins and CPython's json; the examples are also compared with their
twins through the oracle's loops. Then what only the device has: mixed windows with cancelled slots in count mode, PEEK
and ASYNC bursts beside built-in drains, a wrapping ring, B9_ENOSPC, pick's KeyError under retry_for, task-queue and
endpoint-runner callbacks, the SDK mirrors, and a BASELINE-size window of 256-character strings."""
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
from tests import test_gpu_user_handler as G
from tests import test_user_containers_on_host as UC
from tests import test_user_handler_on_host as U
from tests.test_user_containers_on_host import _examples_rules, uc  # noqa: F401  (the host shim and the decline rules)

pytestmark = pytest.mark.gpu
KEY = b"workspace-signing-key"
TQ, ENDPOINT, TF_HTTP_BODY, TF_TASK_MSG = U.TQ, U.ENDPOINT, U.TF_HTTP_BODY, U.TF_TASK_MSG


def new_queue(**kw):
    from beta9_b200.device_queue import DeviceQueue
    if not os.path.exists(B.CONTAINER_CUBIN):
        pytest.fail(f"{B.CONTAINER_CUBIN} is missing: __graft_entry__.build() (beta9_b200.build.build_test_handlers) makes it")
    q = DeviceQueue(**kw)
    q.load_handler(B.CONTAINER_CUBIN, "cscript")
    for name in UC.EXAMPLES + ["echo_str"]:
        q.load_handler(B.EXAMPLE_CUBIN, name)
    return q


@pytest.fixture(scope="module")
def dq():
    q = new_queue(ring_bytes=1 << 30, ring_tasks=1 << 20, max_drain_tasks=1 << 20, max_result_bytes=1 << 30)
    yield q
    q.close()


def device(q, shim):
    """the host shim's signature, answered by one device drain per call; every record must equal the shim's"""
    run = G.device(q)

    def both(payloads, name, rendering, flags=0, ids=None):
        got = run(payloads, name, rendering, flags, ids)
        host = shim(payloads, name, rendering, flags, ids)
        for p, g, h in zip(payloads, got, host):
            assert (g[0], g[1], g[3]) == (h[0], h[1], h[3]), (name, rendering, flags, p, g, h)
        return got
    return both


def sdk_script(ops, rest=UC.REST):
    return json.dumps({"args": [ops] + list(rest), "kwargs": {}}).encode()


def test_scripts(dq, uc):
    run = device(dq, uc)
    UC.check_scripts(run, UC.pair_scripts())
    UC.check_scripts(run, UC.random_scripts(4000, 5))
    for rule, scripts in UC.BROKEN.items():
        for rendering, fl in ((TQ, 0), (ENDPOINT, TF_HTTP_BODY)):
            assert all(g[:2] == (U.UNSUPPORTED, 0) for g in run([sdk_script(s) for s in scripts], "cscript", rendering, fl)), rule


@pytest.mark.parametrize("name", UC.EXAMPLES)
def test_examples(dq, uc, name):
    run = device(dq, uc)
    UC.check_example(run, name, UC.example_payloads(), 0.5)
    UC.check_example(run, name, U.corpus(), 0.8)


def test_examples_mutations(dq, uc):
    run = device(dq, uc)
    base = [b for b in U.corpus() + UC.example_payloads() if len(b) >= 4]
    rng = np.random.default_rng(93)
    alphabet = list(b'{}[],:" 01e.-nulltrackwgsAv\\\x7f\t\nab') + [0xC3, 0xA9, 0xFF, 0x1F]
    bodies = []
    while len(bodies) < 30000:
        m = bytearray(base[int(rng.integers(0, len(base)))])
        pos = int(rng.integers(0, len(m)))
        k = int(rng.integers(0, 3))
        ch = int(rng.choice(alphabet))
        if k == 0: m[pos] = ch
        elif k == 1: del m[pos]
        else: m[pos:pos] = bytes([ch])
        bodies.append(bytes(m))
    for i, name in enumerate(UC.EXAMPLES):
        part = bodies[i::4]
        U.check_tq(run, name, part)
        U.check_ep(run, name, part)


# ---- windows, bursts, rings --------------------------------------------------------------------------------------------
def window(n, seed):
    """n scripts: good containers and values between broken ones, so that a refused writing pass sits beside records"""
    rng = np.random.default_rng(seed)
    good = UC.random_scripts(200, seed)
    bad = [s for ss in UC.BROKEN.values() for s in ss]
    return [bad[int(rng.integers(0, len(bad)))] if rng.random() < 0.3 else good[int(rng.integers(0, len(good)))] for _ in range(n)]


def test_mixed_window_and_cancelled_slots_count_mode(dq, uc):
    scripts = window(1500, 3)
    c = [sdk_script(s) for s in scripts]
    recs, ids = U.records_of(c[:500])
    want = uc(c, "cscript", TQ) + uc(c, "cscript", TQ, TF_HTTP_BODY) + uc(recs, "cscript", TQ, TF_TASK_MSG, ids)
    kinds = [(p, 0, None) for p in c] + [(p, TF_HTTP_BODY, None) for p in c] + [(r, TF_TASK_MSG, i) for r, i in zip(recs, ids)]
    order = np.random.default_rng(5).permutation(len(kinds))
    tids = []
    for k in order:                                                       # one push per task, in the shuffled order
        p, fl, tid = kinds[k]
        tids.append(G.push(dq, [p], fl, [tid] if tid else [int(k + 1_000_000).to_bytes(16, "big")])[0])
    keep = np.ones(len(kinds), bool)
    keep[np.random.default_rng(4).choice(len(kinds), len(kinds) // 3, replace=False)] = False
    dq.cancel(np.stack(tids)[~keep])
    r = dq.drain("cscript")
    assert r.n == int(keep.sum()) and dq.depth() == 0
    got = G.records(r)
    expect = [want[k] for k, kp in zip(order, keep) if kp]
    assert [(g[0], g[1], g[3]) for g in got] == [(w[0], w[1], w[3]) for w in expect]


def test_peek_and_async_beside_built_in_drains(dq, uc):
    c = [U.sdk("w%d x y" % i) for i in range(300)] + [U.sdk({"a": [1, 2]}), U.sdk(""), U.sdk(None)]
    want = {n: [(g[0], g[1], None, g[3]) for g in uc(c, n, TQ)] for n in ("tokens", "describe", "grid")}
    G.push(dq, c)
    dq.drain_launch("identity", peek=True)
    ident = G.records(dq.fetch())
    for _ in range(3):
        for n in ("tokens", "describe"):
            dq.drain_launch(n, peek=True)
            assert G.records(dq.fetch()) == want[n]
        for n in ("tokens", "identity", "describe", "echo_str", "grid"):       # an async burst: the last launch's records wait
            dq.drain_launch(n, peek=True, wait=False)
        assert G.records(dq.fetch()) == want["grid"]
        dq.drain_launch("describe", peek=True, wait=False)
        dq.drain_launch("identity", peek=True, wait=False)
        assert G.records(dq.fetch()) == ident
    assert dq.depth() == len(c)
    dq.drain("tokens")
    G.push(dq, c, TF_HTTP_BODY)
    ep = [(g[0], g[1], None, g[3]) for g in uc(c, "describe", ENDPOINT, TF_HTTP_BODY)]
    dq.drain_launch("tokens", peek=True, endpoint=True, wait=False)
    dq.drain_launch("describe", peek=True, endpoint=True, wait=False)
    assert G.records(dq.fetch()) == ep
    dq.drain("describe", endpoint=True)
    assert dq.depth() == 0


def test_wrapping_ring(uc):
    """a 4 KiB, 32-slot ring: each step pushes a part and drains the part pushed before it"""
    q = new_queue(ring_bytes=4096, ring_tasks=32, max_drain_tasks=32, max_result_bytes=1 << 16)
    try:
        c = [p for p in [sdk_script(s, UC.REST[:8]) for s in window(1600, 11)] if len(p) < 200]
        rng = np.random.default_rng(9)
        pending, i, steps = [], 0, 0
        while i < len(c) or pending:
            if i < len(c):
                k = int(rng.integers(1, 8))
                part = c[i:i + k]
                i += k
                G.push(q, part)
                pending.append(part)
            if len(pending) > 1 or i >= len(c):
                part = pending.pop(0)
                r = q.drain("cscript", max_tasks=len(part))
                assert G.records(r) == [(g[0], g[1], None, g[3]) for g in uc(part, "cscript", TQ)]
                steps += 1
        assert q.depth() == 0 and steps > 100
    finally:
        q.close()


def test_enospc_consumes_nothing(dq):
    c = [U.sdk(" ".join(["word"] * 100))] * 100
    want = json.dumps(["word"] * 100).encode()
    G.push(dq, c)
    dq.drain_launch("tokens")
    with pytest.raises(L.B9Error) as e:
        dq.fetch(cap_bytes=1000)
    assert e.value.code == L.B9_ENOSPC and dq.depth() == 100
    r = dq.fetch()
    assert r.n == 100 and dq.depth() == 0 and all(r.result(i) == want for i in range(100))
    q = new_queue(ring_bytes=1 << 20, ring_tasks=1024, max_drain_tasks=1024, max_result_bytes=4096)
    try:
        G.push(q, c)
        with pytest.raises(L.B9Error) as e:
            q.drain_launch("tokens")
        assert e.value.code == L.B9_ENOSPC and q.depth() == 100
        r = q.drain("tokens", max_tasks=4)
        assert r.n == 4 and q.depth() == 96 and all(r.result(i) == want for i in range(4))
    finally:
        q.close()


def test_pick_key_error_under_retry_for(dq):
    """pick's KeyError is RETRY under retry_for=[KeyError] until the limit, then RETRY_LIMIT; a good pick completes"""
    dq.set_retry_policy([KeyError], 2)
    try:
        c = [U.sdk({"a": 1}, "b"), U.sdk({"a": 1}, "a"), U.sdk({"a": 1}, ["a"])]
        ids = [x.tobytes() for x in G.push(dq, c)]
        seen = []
        for _ in range(4):
            r = dq.drain("pick")
            seen.append([(r.task_ids[i].tobytes(), int(r.status[i]), r.result(i)) for i in range(r.n)])
            if dq.depth() == 0:
                break
        assert seen[0] == [(ids[0], L.ST_RETRY, None), (ids[1], L.ST_COMPLETE, b'{"a": 1}'), (ids[2], L.ST_ERROR, None)], seen
        assert [s[:2] for s in seen[1]] == [(ids[0], L.ST_RETRY)]
        assert [s[:2] for s in seen[2]] == [(ids[0], L.ST_RETRY_LIMIT)] and len(seen) == 3
    finally:
        dq.set_retry_policy([], 0)


def test_callbacks(dq):
    """task queue: the signature over {"data": <the dict or list>}; endpoint runner: D = the text transform of the
    record, signed as {"data": D}, against json.dumps of the twin's result"""
    c = [U.sdk("a b c"), U.sdk({"x": [1, 2.5, None]}), U.sdk(""), U.sdk([]), U.sdk({"a": 1}, "a"), U.sdk("é\U0001F600 \"q\"")]
    dq.set_callback_policy(KEY)
    try:
        for name in ("tokens", "describe", "grid"):
            ids = G.push(dq, c)
            r = dq.drain(name, callbacks=True)
            assert r.n == len(c) and r.cb_timestamp > 0 and np.array_equal(r.task_ids, ids)
            for i in range(r.n):
                st = {0: "COMPLETE", 1: "ERROR", 3: "REJECTED", 4: "UNSUPPORTED"}[int(r.status[i])]
                assert int(r.cb_kind[i]) == CB.callback_kind(st, r.result(i), {}), (name, c[i])
                if int(r.cb_kind[i]) == L.CB_POST:
                    body = CB.callback_body(r.result(i))
                    msg = base64.b64encode(body) + b":%d" % r.cb_timestamp
                    assert r.cb_digest[i].tobytes() == hmac.new(KEY, msg, hashlib.sha256).digest(), (name, c[i])
        dq.set_callback_runners(endpoint=True)
        for name in ("tokens", "describe", "grid"):
            G.push(dq, c, TF_HTTP_BODY)
            r = dq.drain(name, endpoint=True, callbacks=True)
            posted = 0
            for i in range(r.n):
                if int(r.status[i]) != 0:
                    continue
                assert int(r.cb_kind[i]) == L.CB_POST
                args = json.loads(c[i])["args"]
                want = json.dumps(U.twins.TWINS[name](*args))
                body = r.callback_body(i)
                assert body == b'{"data": ' + want.encode() + b"}", (name, c[i], body)
                msg = base64.b64encode(body) + b":%d" % r.cb_timestamp
                assert r.cb_digest[i].tobytes() == hmac.new(KEY, msg, hashlib.sha256).digest()
                posted += 1
            assert posted >= 3
        dq.set_callback_runners()
    finally:
        dq.set_callback_policy(None)


def test_sdk_mirrors():
    from beta9_b200.endpoint import Endpoint
    from beta9_b200.taskqueue import TaskQueue
    tq = TaskQueue(gpu_handler="describe", gpu_handler_image=B.EXAMPLE_CUBIN)
    f = tq(U.twins.describe)
    f.put("x")
    f.put({"b": [1], "a": None})
    f.put()
    f.put(0)
    got = f.process_tasks()
    assert [(t.status, t.result) for t in got] == [("COMPLETE", {"type": "str", "value": "x"}),
                                                   ("COMPLETE", {"type": "dict", "value": {"a": None, "b": [1]}}),
                                                   ("ERROR", None), ("COMPLETE", {"type": "int", "value": 0})], got
    ep = Endpoint(gpu_handler="pick", gpu_handler_image=B.EXAMPLE_CUBIN)(U.twins.pick)
    assert ep.request(b'{"args": [{"a": 1, "\\u00e9": [2]}, "\\u00e9", "a"]}') == (200, '{"é":[2],"a":1}'.encode())
    assert ep.requests([b'{"args": [{"a": 1}, "b"]}', b'{"args": [{"a": 1}]}', b"{"]) == \
        [(500, None), (200, b"{}"), (400, b'{"error":"invalid request payload"}')]


def test_baseline_window_of_strings(dq):
    """configs[1]'s window, 1 Mi SDK payloads of 256-character strings: describe's records are
    {"type": "str", "value": <identity's record>} of the built-in identity drain of the same window; tokens' are
    json.dumps(s.split()) on a sample"""
    n = 1 << 20
    b = synth.strings_batch(n, 256)
    dq.push_batch(b.task_ids, b.payload, b.offsets)
    dq.drain_launch("identity", n, peek=True)
    ident = dq.fetch()
    dq.drain_launch("describe", n, peek=True)
    desc = dq.fetch()
    dq.drain_launch("tokens", n, peek=True)
    tok = dq.fetch()
    assert ident.n == desc.n == tok.n == n
    assert np.all(desc.status == 0) and np.all(tok.status == 0)
    for i in range(n):
        assert desc.result(i) == b'{"type": "str", "value": ' + ident.result(i) + b"}", i
    for i in np.random.default_rng(1).choice(n, 20000, replace=False):
        s = go_unmarshal_task_payload(b.payload[int(b.offsets[i]):int(b.offsets[i + 1])].tobytes())[0][0]   # (as Go decoded it)
        assert tok.result(int(i)) == (json.dumps(s.split()).encode() if s.split() else None), i
    dq.drain("identity", n)
    assert dq.depth() == 0
