"""GPU tests of the callback pass (b9_set_callback_policy / b9_drain_fetch_callbacks): every record's callback kind equals
the oracle's restatement of send_callback (oracle/pyoracle/callback.py), and every B9_CB_POST digest equals
hmac(key, base64(body) + b":%d" % timestamp) with the body built from the record."""
import base64
import hashlib
import hmac
import json
import uuid

import numpy as np
import pytest

from beta9_b200 import _lib as L
from beta9_b200 import synth
from beta9_b200.device_queue import STATUS_NAMES, DeviceQueue
from oracle.pyoracle import callback as cb
from oracle.pyoracle.loop import sdk_put_payload
from tests.golden.make_ref_callback_golden import explicit_wires
from tests.golden.make_ref_retry_golden import corpus_wires
from tests.pickle_corpus import frame_one

pytestmark = pytest.mark.gpu
HANDLERS = ["identity", "crc32", "vadd_f32", "json_sum"]
KEY = b"workspace-signing-key-0123456789"


def queue(**kw):
    o = dict(ring_bytes=1 << 24, ring_tasks=1 << 14, max_drain_tasks=1 << 14, max_result_bytes=1 << 24)
    o.update(kw)
    return DeviceQueue(**o)


def ids_for(n, salt):
    return np.frombuffer(b"".join(uuid.UUID(int=(salt << 64) | (i + 1)).bytes for i in range(n)), np.uint8).reshape(n, 16)


def push(q, payloads, ids, flags=None, retries=None):
    off = np.zeros(len(payloads) + 1, np.uint64)
    np.cumsum([len(p) for p in payloads], out=off[1:])
    q.push_batch(ids, np.frombuffer(b"".join(payloads), np.uint8), off, flags=flags, retries=retries)


def expected_kind(status, result, cb_kwarg=False, pickle=False):
    return cb.callback_kind(status, result, {"callback_url": 1} if cb_kwarg else {}, pickle=pickle)


def check(res, key, cb_kwarg_ids=(), pickle_ids=(), sample=None):
    """Kinds against the oracle from each record's own status and bytes, digests against hmac; -> kinds seen."""
    assert res.cb_kind is not None and res.cb_kind.shape[0] == res.n
    if key:
        assert res.cb_timestamp > 1_700_000_000
    else:
        assert res.cb_timestamp == 0
    idx = range(res.n) if sample is None else sorted(set(np.random.default_rng(5).integers(0, res.n, sample).tolist()))
    seen = set()
    for i in idx:
        rid = res.task_ids[i].tobytes()
        st = STATUS_NAMES[int(res.status[i])]
        want = expected_kind(st, res.result(i), rid in cb_kwarg_ids, rid in pickle_ids)
        assert int(res.cb_kind[i]) == want, (i, st, res.result(i), int(res.cb_kind[i]), want)
        seen.add(want)
        d = res.cb_digest[i].tobytes()
        if want == cb.CB_POST and key:
            assert d == hmac.new(key, cb.sign_message(res.callback_body(i), res.cb_timestamp), hashlib.sha256).digest(), i
        else:
            assert d == bytes(32), i
    return seen


def mixed_corpus(salt):
    """Valid and failing tasks of every framing: SDK payloads, HTTP bodies, TaskMessage records, callback_url kwargs,
    pickle and UNSUPPORTED tasks and REJECTED payloads. -> payloads, ids, flags, ids with a callback_url kwarg, pickle ids"""
    from oracle.pyoracle import loop
    p, f, has_cb = [], [], []
    for a, kw in [(("hello",), {}), (("",), {}), ((3,), {}), (({"values": [1, 2, 3]},), {}), (({"values": [1e308, 1e308]},), {}),
                  (({"values": [-1e308, -1e308]},), {}), (("AACAPwAAAEAAAIA/AAAAQA==",), {}), ((), {}), (("x", "y"), {}),
                  (("x",), {"callback_url": "http://o"}), (("x",), {"callback_url": ""}), (("x",), {"callback_url": None}),
                  (("x",), {"k": 1}), (([1, [2, {"a": "é"}]],), {})]:
        p.append(sdk_put_payload(*a, **kw)); f.append(0); has_cb.append("callback_url" in kw)
        p.append(json.dumps({"args": list(a), **({"kwargs": kw} if kw else {})}).encode()); f.append(L.TF_HTTP_BODY); has_cb.append("callback_url" in kw)
    p += [b'{"args": ["x"], "callback_url": "u"}', b'{"args": ["x"], "kwargs": {"callback\\u005furl": 1}}', b"not json", b"[1]",
          b'{"args": [' + b"[" * 20 + b"]" * 20 + b']}', b'{"args": [1e999]}']
    f += [L.TF_HTTP_BODY, 0, 0, 0, 0, 0]
    has_cb += [True, True, False, False, False, False]
    n0 = len(p)
    ids = ids_for(n0 + 6, salt)
    calls = [(("rec",), {}), (("r",), {"callback_url": "u"}), (({"values": [4]},), {})]
    for w in loop.run_task_loop([sdk_put_payload(*a, **k) for a, k in calls], [bytes(ids[n0 + i]) for i in range(3)], "identity", keep_wire=True):
        p.append(w.wire); f.append(L.TF_TASK_MSG)
    has_cb += [False, True, False]
    p += [frame_one({"args": ["s"], "kwargs": {}}), frame_one({"args": [{"values": [1]}], "kwargs": {}}), frame_one(5)]
    f += [L.TF_PICKLE] * 3
    has_cb += [False] * 3
    cbs = {bytes(ids[i]) for i in range(len(p)) if has_cb[i]}
    pk = {bytes(ids[i]) for i in range(len(p)) if f[i] == L.TF_PICKLE}
    return p, ids[:len(p)], np.array(f, np.uint8), cbs, pk


@pytest.mark.parametrize("handler", HANDLERS)
@pytest.mark.parametrize("key_len", [0, 1, 64, 65, 200])
def test_mixed_corpus_every_key_length(handler, key_len):
    key = bytes((i * 13 + 5) & 0xFF for i in range(key_len))
    p, ids, flags, cbs, pk = mixed_corpus(1)
    with queue() as q:
        q.set_callback_policy(key)
        push(q, p, ids, flags)
        r = q.drain(handler, callbacks=True)
        assert r.n == len(p)
        seen = check(r, key, cbs, pk)
        assert {cb.CB_POST, cb.CB_HOST, cb.CB_NONE} <= seen
        if handler == "json_sum":
            assert cb.CB_UNSENDABLE in seen


@pytest.mark.parametrize("handler", HANDLERS)
def test_golden_corpus_records(handler):
    """The reference runner's corpus as TaskMessage records: kinds equal the oracle's for the statuses the runner reported."""
    wires = corpus_wires(handler) + explicit_wires(handler)
    ids = np.frombuffer(b"".join(uuid.UUID(json.loads(w)["task_id"]).bytes for w in wires), np.uint8).reshape(-1, 16)
    cbs = {bytes(ids[i]) for i, w in enumerate(wires) if "callback_url" in (json.loads(w)["kwargs"] or {})}
    with queue() as q:
        q.set_callback_policy(KEY)
        push(q, wires, ids, np.full(len(wires), L.TF_TASK_MSG, np.uint8))
        r = q.drain(handler, callbacks=True)
        assert r.n == len(wires)
        check(r, KEY, cbs)


BASELINE = {"identity": lambda: synth.strings_batch(1 << 20, 256), "crc32": lambda: synth.crc_batch(1 << 20),
            "vadd_f32": lambda: synth.vadd_batch(1_250_000), "json_sum": lambda: synth.json_batch(25_000)}


@pytest.mark.parametrize("handler", HANDLERS)
def test_baseline_size(handler):
    """At the BASELINE size per GPU: the records are the same with and without the policy, every kind follows the
    record's status, and a sample of the digests equals hmac."""
    b = BASELINE[handler]()
    with DeviceQueue(ring_bytes=1 << 31, ring_tasks=1 << 21, max_drain_tasks=1 << 21, max_result_bytes=1 << 31) as q:
        q.push_batch(b.task_ids, b.payload, b.offsets)
        q.drain_launch(handler, b.n, peek=True)
        plain = q.fetch(cap_tasks=b.n)
        q.set_callback_policy(KEY)
        q.drain_launch(handler, b.n, peek=True)
        r = q.fetch(cap_tasks=b.n, callbacks=True)
        assert r.n == plain.n == b.n
        assert np.array_equal(r.status, plain.status) and np.array_equal(r.has_result, plain.has_result)
        assert np.array_equal(r.fifo_payload(), plain.fifo_payload())
        post = (r.status == L.ST_COMPLETE) | (r.status == L.ST_ERROR)
        assert np.all(r.cb_kind[post & (r.cb_kind != L.CB_UNSENDABLE)] == L.CB_POST)
        assert np.all(r.cb_kind[r.status == L.ST_UNSUPPORTED] == L.CB_HOST)
        check(r, KEY, sample=20_000)


def test_long_records():
    """Records of 64 KiB and more, and one multi-MiB vadd_f32 record (thousands of compressions on one lane)."""
    floats = np.arange(1 << 18, dtype=np.float32)
    vec = base64.b64encode(floats.tobytes() + (floats * 2).tobytes()).decode()
    with queue(ring_bytes=1 << 26, max_result_bytes=1 << 26, max_task_bytes=1 << 24) as q:
        q.set_callback_policy(KEY)
        push(q, [sdk_put_payload("x" * 70000), sdk_put_payload("y" * 300000), sdk_put_payload("z")], ids_for(3, 2))
        r = q.drain("identity", callbacks=True)
        assert [len(r.result(i)) for i in range(3)] == [70002, 300002, 3]
        check(r, KEY)
        push(q, [sdk_put_payload(vec)], ids_for(1, 3))
        r = q.drain("vadd_f32", callbacks=True)
        assert r.n == 1 and r.status[0] == L.ST_COMPLETE and len(r.result(0)) > 1 << 20
        check(r, KEY)


def test_cancelled_slots_and_retry_policy():
    """A window with cancelled slots (records compacted: the count pre-pass's prefixes map them), and RETRY / RETRY_LIMIT
    under a retry policy, which the runner never calls back for."""
    p, ids, flags, cbs, pk = mixed_corpus(4)
    rng = np.random.default_rng(4)
    reps = 40
    P = p * reps
    I = ids_for(len(P), 5)
    F = np.tile(flags, reps)
    cbs = {bytes(I[i]) for i in range(len(P)) if bytes(ids[i % len(p)]) in cbs}
    pk = {bytes(I[i]) for i in range(len(P)) if F[i] == L.TF_PICKLE}
    F = F | np.where(rng.random(len(P)) < 0.2, L.TF_CANCELLED, 0).astype(np.uint8)
    retries = rng.integers(0, 3, len(P)).astype(np.uint8)
    with queue() as q:
        q.set_callback_policy(KEY)
        q.set_retry_policy([TypeError], 1)
        push(q, P, I, F, retries)
        r = q.drain("crc32", callbacks=True)
        assert r.n == int(np.sum((F & L.TF_CANCELLED) == 0))
        st = set(r.status.tolist())
        assert L.ST_RETRY in st and L.ST_RETRY_LIMIT in st
        check(r, KEY, cbs, pk)
        assert np.all(r.cb_kind[(r.status == L.ST_RETRY) | (r.status == L.ST_RETRY_LIMIT)] == L.CB_NONE)


def test_peek_async_burst_small_ring_and_enospc():
    p, ids, flags, cbs, pk = mixed_corpus(6)
    with queue(ring_bytes=1 << 12, ring_tasks=64, max_drain_tasks=64, max_result_bytes=1 << 16) as q:
        q.set_callback_policy(KEY)
        for rnd in range(6):                            # a small ring: the windows wrap it
            sel = list(range(rnd % 3, len(p), 3))
            push(q, [p[i] for i in sel], ids[sel], flags[sel])
            q.drain_launch("identity", 1 << 20, peek=True)
            a = q.fetch(callbacks=True, cap_tasks=64)
            check(a, KEY, cbs, pk)
            for _ in range(3):                          # a burst of async launches keeps the last one's callbacks
                q.drain_launch("identity", 1 << 20, peek=True, wait=False)
            b = q.fetch(callbacks=True, cap_tasks=64)
            assert np.array_equal(a.cb_kind, b.cb_kind) and np.array_equal(a.status, b.status)
            check(b, KEY, cbs, pk)
            q.drain_launch("identity", 1 << 20)
            st = q.stats()
            small = L.Results(*([0] * 6), 1, 1 << 20, 0, 0, 0, 0, 0.0, 0)
            kind = np.zeros(1, np.uint8); dg = np.zeros((1, 32), np.uint8)
            rc = q._lib.b9_drain_fetch_callbacks(q._ctx, small, L.Callbacks(kind.ctypes.data, dg.ctypes.data, 1, 0))
            assert rc == L.B9_ENOSPC and q.depth() == len(sel)
            c = q.fetch(callbacks=True, cap_tasks=64)
            assert c.n == len(sel) and q.depth() == 0 and st.drains >= 1
            check(c, KEY, cbs, pk)


def test_einval_without_policy_and_after_endpoint_launch():
    p, ids, flags, cbs, pk = mixed_corpus(7)
    with queue() as q:
        push(q, p, ids, flags)
        q.drain_launch("identity", 1 << 20, peek=True)
        with pytest.raises(L.B9Error) as e:
            q.fetch(callbacks=True)
        assert e.value.code == L.B9_EINVAL
        q.set_callback_policy(b"")
        q.drain_launch("identity", 1 << 20, peek=True, endpoint=True)
        with pytest.raises(L.B9Error) as e:
            q.fetch(callbacks=True)
        assert e.value.code == L.B9_EINVAL
        q.drain_launch("identity", 1 << 20, peek=True)
        check(q.fetch(callbacks=True), b"", cbs, pk)
        q.set_callback_policy(None)
        q.drain_launch("identity", 1 << 20, peek=True)
        with pytest.raises(L.B9Error):
            q.fetch(callbacks=True)


def test_sdk_mirror_task_callback():
    from beta9_b200.taskqueue import TaskQueue
    tq = TaskQueue(callback_url="http://cb.invalid/hook", signing_key=KEY, gpu_handler="json_sum", max_pending_tasks=1000)
    w = tq(lambda obj: sum(obj["values"]))
    calls = [(({"values": [1, 2]},), {}), (({"values": []},), {}), (({"values": [1e308, 1e308]},), {}), (("x",), {}),
             (({"values": [1]},), {"callback_url": "http://override.invalid/x"}), (({"values": [1]},), {"callback_url": ""})]
    tasks = w.put_batch(calls)
    done = {t.id: t for t in w.process_tasks()}
    for t, (a, kw) in zip(tasks, calls):
        d = done[t.id]
        want = cb.runner_callback(uuid.UUID(t.id).bytes, d.status, d.result_bytes, kw, "http://cb.invalid/hook", KEY,
                                  int(d.callback[2]["X-Task-Timestamp"]) if d.callback else 0)
        assert d.callback == want, (a, kw, d.callback, want)
    assert sum(1 for t in done.values() if t.callback is None) == 1          # the non-finite total: requests refuses it
