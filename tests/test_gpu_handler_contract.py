"""GPU tests of the user-handler header's contract: the test-only handlers of tests/handlers, loaded from the cubin build()
makes (tests/handlers/contract.cubin), drained on the device over the corpora of tests/test_handler_contract_on_host.py.
Every record must equal the host shim's and the twin's expectation. Then what only the device has: broken scripts
between good records of one warp-tile (a refused overrun must leave its neighbours' bytes alone), odd windows, cancelled
slots, a wrapping ring, B9_ENOSPC, the retry policy for each exception class, callbacks, and both handler forms loaded
side by side with peek and async bursts next to a built-in drain."""
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
from tests import test_handler_contract_on_host as H
from tests.handlers import contract_twins as T
from tests.test_handler_contract_on_host import ct  # noqa: F401  (the host shim, as a fixture)

pytestmark = pytest.mark.gpu
NAMES = H.NAMES
KEY = b"workspace-signing-key"
TQ, ENDPOINT, TF_HTTP_BODY = H.TQ, H.ENDPOINT, H.TF_HTTP_BODY
S, E = H.op(T.STR_BEGIN), H.op(T.STR_END)


def new_queue(**kw):
    from beta9_b200.device_queue import DeviceQueue
    if not os.path.exists(B.TEST_CUBIN):
        pytest.fail(f"{B.TEST_CUBIN} is missing: __graft_entry__.build() (beta9_b200.build.build_test_handlers) makes it")
    q = DeviceQueue(**kw)
    for name in NAMES:
        q.load_handler(B.TEST_CUBIN, name)
    return q


@pytest.fixture(scope="module")
def dq():
    q = new_queue(ring_bytes=1 << 28, ring_tasks=1 << 18, max_drain_tasks=1 << 17, max_result_bytes=1 << 28)
    yield q
    q.close()


def records(r):
    return [(int(r.status[i]), int(r.has_result[i]), None, r.result(i) or b"") for i in range(r.n)]


def push(q, payloads, flags=0, ids=None):
    b = synth.from_payloads(list(payloads))
    tid = b.task_ids if ids is None else np.frombuffer(b"".join(ids), np.uint8).reshape(-1, 16)
    q.push_batch(tid, b.payload, b.offsets, flags=np.full(b.n, flags, np.uint8))
    return tid


def device(q, shim):
    """the host shim's signature, answered by one device drain per call; every record must also equal the shim's"""
    def run(payloads, name, rendering, flags=0, ids=None):
        if not payloads:
            return []
        assert q.depth() == 0
        push(q, payloads, flags, ids)
        r = q.drain(name, endpoint=rendering == ENDPOINT)
        assert r.n == len(payloads) and q.depth() == 0
        got = records(r)
        host = shim(payloads, name, rendering, flags, ids)
        for p, g, h in zip(payloads, got, host):
            assert (g[0], g[1], g[3]) == (h[0], h[1], h[3]), (name, rendering, flags, p, g, h)
        return got
    return run


def test_scripts(dq, ct):
    run = device(dq, ct)
    H.check_scripts(run, H.pair_scripts())
    H.check_scripts(run, H.edge_scripts())
    H.check_scripts(run, H.random_scripts(3000, 7))


def test_inspect(dq, ct):
    run = device(dq, ct)
    H.check_inspect(run, "inspect", H.value_payloads())
    H.check_inspect(run, "inspect", H.key_payloads(), min_share=0.8)
    H.check_inspect(run, "inspect_keys", H.inspect_keys_payloads(), min_share=0.8)


# ---- broken scripts between good ones ------------------------------------------------------------------------------------
A = H.op(T.CP, 0x41)
BROKEN = [
    [S, A, H.op(T.CP_WRITE, 0x41), E],                  # the writing pass one byte longer: its closing quote is past the end
    [S, A, H.op(T.CP_WRITE, 0x1F600), E],               # ... many bytes longer
    [S, A, H.op(T.CP_COUNT, 0x41), E],                  # shorter
    [S, H.op(T.CP_COUNT, 0xE9), H.op(T.CP_WRITE, 0xD800), E],   # as long, with a surrogate (task queue)
    [S, H.op(T.CP_COUNT, 0x800), H.op(T.CP_WRITE, 0xDC00), E],  # as long, with a surrogate (endpoint)
    [H.op(T.INT, 1), H.op(T.INT, 2)], [S, A], [A], [S, H.op(T.CP, 0xD800), E], [S, H.op(T.CP, 0x110000), E], [],
    [H.op(T.RETURN, 3)], [H.op(T.RETURN, 0x40)], [H.op(T.RETURN, -2)], [S, A, E, H.op(T.RETURN, 0x21)],
]
GOOD = [[H.op(T.INT, 12345)], [H.op(T.BOOL, 0)], [H.op(T.NONE)], [H.op(T.REAL, H.bits(2.5))], [S, A, E],
        [S] + [H.op(T.CP, 0x61 + k % 26) for k in range(13)] + [E], [S, H.op(T.CP, 0x1F600), H.op(T.CP, 0x22), E], [H.op(T.BOOL, 1)],
        [H.op(T.INT, -7)]]


def tile_window(n, seed):
    """n scripts: each broken one followed by a scalar record (whose bytes an overrun would land on) and string records"""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        out.append(BROKEN[int(rng.integers(0, len(BROKEN)))])
        out.append(GOOD[int(rng.integers(0, 4))] if rng.random() < 0.7 else GOOD[0])
        out += [GOOD[int(rng.integers(0, len(GOOD)))] for _ in range(int(rng.integers(0, 3)))]
    return out[:n]


def want_of(scripts, rendering, flags, ct):
    """the records of the scripts: the shim's, which the host tests pin to the twin"""
    return [(g[0], g[1], None, g[3]) for g in ct([H.sdk(s) for s in scripts], "script", rendering, flags)]


@pytest.mark.parametrize("name", ["script", "script_sig"])
def test_broken_scripts_between_good_ones(dq, ct, name):
    for n in (1, 31, 33, 97, 1001):
        scripts = tile_window(n, n)
        for rendering, flags in ((TQ, 0), (ENDPOINT, TF_HTTP_BODY)):
            push(dq, [H.sdk(s) for s in scripts], flags)
            got = records(dq.drain(name, endpoint=rendering == ENDPOINT))
            assert got == want_of(scripts, rendering, flags, ct), (n, rendering)
            assert any(g[0] == H.UNSUPPORTED for g in got) and (n == 1 or any(g[1] for g in got))


@pytest.mark.parametrize("name", ["script", "script_sig"])
def test_cancelled_slots_count_mode(dq, ct, name):
    scripts = tile_window(777, 3)
    want = want_of(scripts, TQ, 0, ct)
    ids = push(dq, [H.sdk(s) for s in scripts])
    keep = np.ones(len(scripts), bool)
    keep[np.random.default_rng(4).choice(len(scripts), 111, replace=False)] = False
    dq.cancel(ids[~keep])
    r = dq.drain(name)
    assert r.n == int(keep.sum()) and r.n_popped == len(scripts)
    assert records(r) == [want[i] for i in np.flatnonzero(keep)]
    assert np.array_equal(r.task_ids, ids[keep])


def test_wrapping_ring(ct):
    """a 4 KiB, 32-slot ring: each step pushes a part and drains the part pushed before it, so that windows wrap both the
    slots and the bytes"""
    q = new_queue(ring_bytes=4096, ring_tasks=32, max_drain_tasks=32, max_result_bytes=1 << 16)
    try:
        scripts = tile_window(700, 5)
        rng = np.random.default_rng(9)
        pending, i, steps = [], 0, 0
        while i < len(scripts) or pending:
            if i < len(scripts):
                k = int(rng.integers(1, 8))
                part = scripts[i:i + k]
                i += k
                push(q, [H.sdk(s) for s in part])
                pending.append(part)
            if len(pending) > 1 or i >= len(scripts):
                part = pending.pop(0)
                name = ("script", "script_sig")[steps % 2]
                r = q.drain(name, max_tasks=len(part))
                assert records(r) == want_of(part, TQ, 0, ct)
                steps += 1
        assert q.depth() == 0 and steps > 100
    finally:
        q.close()


def test_enospc_consumes_nothing(dq):
    s = [S] + [H.op(T.CP, 0x78)] * 300 + [E]
    c = [H.sdk(s)] * 100
    push(dq, c)
    dq.drain_launch("script")
    assert dq.running() == 100
    with pytest.raises(L.B9Error) as e:
        dq.fetch(cap_bytes=1000)
    assert e.value.code == L.B9_ENOSPC and dq.depth() == 100
    r = dq.fetch()
    assert r.n == 100 and dq.depth() == 0 and r.result(99) == json.dumps("x" * 300).encode()
    q = new_queue(ring_bytes=1 << 20, ring_tasks=1024, max_drain_tasks=1024, max_result_bytes=4096)
    try:
        push(q, c)
        with pytest.raises(L.B9Error) as e:
            q.drain_launch("script_sig")
        assert e.value.code == L.B9_ENOSPC and q.depth() == 100
        r = q.drain("script_sig", max_tasks=10)
        assert r.n == 10 and q.depth() == 90 and all(r.result(i) == json.dumps("x" * 300).encode() for i in range(10))
    finally:
        q.close()


@pytest.mark.parametrize("bit", sorted(T.EXC_CLASSES))
def test_retry_policy_for_each_class(dq, bit):
    """a single-bit return is RETRY until the limit, then RETRY_LIMIT; a multi-bit or unknown return stays UNSUPPORTED and
    is never retried; a good script completes"""
    dq.set_retry_policy([T.EXC_CLASSES[bit]], 2)
    try:
        for name in ("script", "script_sig"):
            c = [H.sdk([H.op(T.RETURN, bit)]), H.sdk([H.op(T.INT, 5)]), H.sdk([H.op(T.RETURN, bit | 0x40 if bit == 1 else bit | 1)]),
                 H.sdk([H.op(T.RETURN, 0x40)]), H.sdk([H.op(T.RETURN, -2)]), H.sdk([S, A, E, H.op(T.RETURN, bit)])]
            ids = push(dq, c)
            seen = []
            for _ in range(4):
                r = dq.drain(name)
                seen.append([(r.task_ids[i].tobytes(), int(r.status[i])) for i in range(r.n)])
                if dq.depth() == 0:
                    break
            t = [x.tobytes() for x in ids]
            assert seen[0] == [(t[0], L.ST_RETRY), (t[1], L.ST_COMPLETE), (t[2], L.ST_UNSUPPORTED), (t[3], L.ST_UNSUPPORTED),
                               (t[4], L.ST_UNSUPPORTED), (t[5], L.ST_RETRY)], (name, seen)
            assert seen[1] == [(t[0], L.ST_RETRY), (t[5], L.ST_RETRY)]
            assert seen[2] == [(t[0], L.ST_RETRY_LIMIT), (t[5], L.ST_RETRY_LIMIT)] and len(seen) == 3
        # another class than the policy's stays ERROR
        other = 0x01 if bit != 0x01 else 0x02
        push(dq, [H.sdk([H.op(T.RETURN, other)])])
        assert int(dq.drain("script").status[0]) == L.ST_ERROR and dq.depth() == 0
    finally:
        dq.set_retry_policy([], 0)


CALLBACK_SCRIPTS = [[H.op(T.NONE)], [H.op(T.BOOL, 0)], [H.op(T.BOOL, 1)], [H.op(T.INT, 0)], [H.op(T.INT, -3)], [S, E],
                    [H.op(T.REAL, 0x8000000000000000)], [H.op(T.REAL, 0x7FF8000000000000)], [H.op(T.REAL, 0xFFF8000000000001)],
                    [H.op(T.REAL, 0x7FF0000000000000)], [H.op(T.REAL, 0xFFF0000000000000)], [H.op(T.REAL, H.bits(0.1))],
                    [S, A, E], [S, H.op(T.CP, 0xE9), H.op(T.CP, 0x1F600), H.op(T.CP, 0x22), H.op(T.CP, 0x0A), E],
                    [H.op(T.RETURN, 0x10)], [H.op(T.RETURN, 3)], [S, A, H.op(T.CP_WRITE, 0x41), E]]


def test_callbacks(dq):
    c = [H.sdk(s) for s in CALLBACK_SCRIPTS]
    dq.set_callback_policy(KEY)
    try:
        for name in ("script", "script_sig"):
            ids = push(dq, c)
            r = dq.drain(name, callbacks=True)
            assert r.n == len(c) and r.cb_timestamp > 0 and np.array_equal(r.task_ids, ids)
            for i in range(r.n):
                st = {0: "COMPLETE", 1: "ERROR", 3: "REJECTED", 4: "UNSUPPORTED"}[int(r.status[i])]
                assert int(r.cb_kind[i]) == CB.callback_kind(st, r.result(i), {}), (name, CALLBACK_SCRIPTS[i])
                if int(r.cb_kind[i]) == L.CB_POST:
                    sig, _ = CB.sign_payload(CB.callback_body(r.result(i)), KEY, r.cb_timestamp)
                    assert r.cb_digest[i].tobytes().hex() == sig
        # the endpoint runner's: D = json.dumps of the response value, signed as {"data": D}
        dq.set_callback_runners(endpoint=True)
        for name in ("script", "script_sig"):
            push(dq, c, TF_HTTP_BODY)
            r = dq.drain(name, endpoint=True, callbacks=True)
            for i in range(r.n):
                st = int(r.status[i])
                want = L.CB_POST if st == 0 else L.CB_NONE if st == L.ST_REJECTED else L.CB_HOST
                assert int(r.cb_kind[i]) == want, (name, CALLBACK_SCRIPTS[i])
                if want == L.CB_POST:
                    body = r.callback_body(i)
                    assert body == b'{"data": ' + json.dumps(json.loads(r.result(i))).encode() + b"}"
                    msg = base64.b64encode(body) + b":%d" % r.cb_timestamp
                    assert r.cb_digest[i].tobytes() == hmac.new(KEY, msg, hashlib.sha256).digest()
        dq.set_callback_runners()
    finally:
        dq.set_callback_policy(None)


def test_both_forms_with_bursts_beside_a_built_in_drain(dq, ct):
    scripts = H.pair_scripts()[::3]
    c = [H.sdk(s) for s in scripts]
    want = {n: want_of(scripts, TQ, 0, ct) for n in ("script", "script_sig")}
    push(dq, c)
    dq.drain_launch("identity", peek=True)
    ident = records(dq.fetch())
    for rnd in range(3):
        for n in NAMES[:2]:
            dq.drain_launch(n, peek=True)
            assert records(dq.fetch()) == want[n]
        for n in ["script", "identity", "script_sig", "inspect", "script"]:     # an async burst: the last launch's records wait
            dq.drain_launch(n, peek=True, wait=False)
        assert records(dq.fetch()) == want["script"]
        dq.drain_launch("script_sig", peek=True, wait=False)
        dq.drain_launch("identity", peek=True, wait=False)
        assert records(dq.fetch()) == ident
    assert dq.depth() == len(c)
    dq.drain("script_sig")
    push(dq, c, TF_HTTP_BODY)
    ep = want_of(scripts, ENDPOINT, TF_HTTP_BODY, ct)
    dq.drain_launch("script", peek=True, endpoint=True, wait=False)
    dq.drain_launch("script_sig", peek=True, endpoint=True, wait=False)
    assert records(dq.fetch()) == ep
    dq.drain("script", endpoint=True)
    assert dq.depth() == 0
