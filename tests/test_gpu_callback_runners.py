"""GPU tests of the runners' callback passes (b9_set_callback_runners / b9_drain_fetch_callback_requests): every record's
kind, callback JSON D and URL equal the oracle's restatement of the function and endpoint runners' send_callback
(tests/callback_runners_oracle.py), and every B9_CB_POST digest equals hmac(key, base64({"data": D}) + b":%d" % timestamp)."""
import hashlib
import hmac
import json
import uuid

import cloudpickle
import numpy as np
import pytest

from beta9_b200 import _lib as L
from beta9_b200 import synth
from beta9_b200.device_queue import STATUS_NAMES, DeviceQueue
from oracle.pyoracle import callback as cb0
from tests import callback_runners_oracle as cb
from oracle.pyoracle import funcloop
from tests.pickle_corpus import frame_one, structured_blobs

pytestmark = pytest.mark.gpu
HANDLERS = ["identity", "crc32", "vadd_f32", "json_sum"]
KEYS = [b"", b"k", b"K" * 64, b"L" * 65, b"M" * 200]


def queue(**kw):
    o = dict(ring_bytes=1 << 26, ring_tasks=1 << 15, max_drain_tasks=1 << 15, max_result_bytes=1 << 27)
    o.update(kw)
    return DeviceQueue(**o)


def ids_for(n, salt):
    return np.frombuffer(b"".join(uuid.UUID(int=(salt << 64) | (i + 1)).bytes for i in range(n)), np.uint8).reshape(n, 16)


def push(q, payloads, ids, flags):
    off = np.zeros(len(payloads) + 1, np.uint64)
    np.cumsum([len(p) for p in payloads], out=off[1:])
    q.push_batch(ids, np.frombuffer(b"".join(payloads), np.uint8), off, flags=np.asarray(flags, np.uint8))


def function_blobs():
    blobs = structured_blobs()
    for url in (None, "", 0, "http://x", b"http://x", 5, "http://é"):
        blobs.append(funcloop.frame_call("s", callback_url=url))
    for v in (b"x", {b"k": 1}, float("nan"), {1.5: 1, float("inf"): 2}, "\x7f\xe9€\U0001F600\ud800", 2 ** 63, [[1, "a"]] * 3, None, ""):
        blobs.append(frame_one(v))
    return blobs


def expected(res, i, kind_of_payload):
    """(kind, D, url) the oracle gives record i; kind_of_payload: id -> ("fn", blob) / ("ep", body) / ("tq", None)"""
    st = STATUS_NAMES[int(res.status[i])]
    what, blob = kind_of_payload[res.task_ids[i].tobytes()]
    if what == "fn":
        if st != "COMPLETE":
            return cb.CB_HOST, None, None
        kw = funcloop.load_args(blob).get("kwargs") or {}
        return cb.function_callback(st, cloudpickle.loads(res.result(i)), kw)
    if what == "ep":
        k, d = cb.endpoint_callback(st, res.result(i))
        return k, d, None
    k = cb0.callback_kind(st, res.result(i))
    return k, (res.result(i) or b"{}") if k == cb.CB_POST else None, None


def check(res, key, kind_of_payload):
    assert res.cb_body_len is not None and res.cb_kind.shape[0] == res.n
    seen = set()
    for i in range(res.n):
        k, d, url = expected(res, i, kind_of_payload)
        assert int(res.cb_kind[i]) == k, (i, STATUS_NAMES[int(res.status[i])], res.result(i), int(res.cb_kind[i]), k)
        seen.add(k)
        if k == cb.CB_POST:
            assert res.callback_body(i) == cb0.BODY_PREFIX + d + b"}", i
            assert res.callback_url(i) == url, i
        dg = res.cb_digest[i].tobytes()
        if k == cb.CB_POST and key:
            assert dg == hmac.new(key, cb0.sign_message(res.callback_body(i), res.cb_timestamp), hashlib.sha256).digest(), i
        else:
            assert dg == bytes(32), i
    return seen


@pytest.mark.parametrize("handler", HANDLERS)
@pytest.mark.parametrize("key", KEYS, ids=lambda k: f"key{len(k)}")
def test_function_runner(handler, key):
    blobs = function_blobs()
    q = queue()
    q.set_callback_policy(key)
    q.set_callback_runners(function=True)
    ids = ids_for(len(blobs), 1)
    push(q, blobs, ids, [L.TF_PICKLE] * len(blobs))
    m = {ids[i].tobytes(): ("fn", b) for i, b in enumerate(blobs)}
    res = q.drain(handler, full_pickle=True, callbacks=True)
    assert res.n == len(blobs)
    seen = check(res, key, m)
    assert cb.CB_POST in seen and cb.CB_HOST in seen
    if handler == "identity":
        assert cb.CB_UNSENDABLE in seen
        assert any(res.callback_url(i) == "http://x" for i in range(res.n))
    q.close()


def endpoint_bodies():
    from tests.golden.make_ref_endpoint_golden import bodies
    return bodies()


@pytest.mark.parametrize("handler", HANDLERS)
@pytest.mark.parametrize("key", KEYS, ids=lambda k: f"key{len(k)}")
def test_endpoint_runner(handler, key):
    bodies = endpoint_bodies()
    q = queue()
    q.set_callback_policy(key)
    q.set_callback_runners(endpoint=True)
    ids = ids_for(len(bodies), 2)
    push(q, bodies, ids, [L.TF_HTTP_BODY] * len(bodies))
    m = {ids[i].tobytes(): ("ep", b) for i, b in enumerate(bodies)}
    res = q.drain(handler, endpoint=True, callbacks=True)
    assert res.n == len(bodies)
    seen = check(res, key, m)
    assert cb.CB_POST in seen and cb.CB_NONE in seen
    q.close()


def test_mixed_window_cancelled_peek_async_and_wrap():
    """Task-queue and pickle tasks in one window with cancelled slots (count mode), a PEEK launch, an ASYNC burst, and a
    small ring that wraps."""
    key = b"workspace"
    q = queue(ring_bytes=1 << 20, ring_tasks=1 << 10, max_drain_tasks=1 << 10, max_result_bytes=1 << 22)
    q.set_callback_policy(key)
    q.set_callback_runners(function=True, endpoint=True)
    fn = function_blobs()[:150]
    tq = [b'{"args": ["x%d"], "kwargs": {}}' % i for i in range(150)]
    salt = 10
    for rnd in range(6):
        payloads, flags, m = [], [], {}
        for i in range(150):
            payloads += [fn[(i + rnd) % len(fn)], tq[i]]
            flags += [L.TF_PICKLE, 0]
        ids = ids_for(len(payloads), salt)
        salt += 1
        for i, p in enumerate(payloads):
            m[ids[i].tobytes()] = ("fn", p) if flags[i] == L.TF_PICKLE else ("tq", None)
        push(q, payloads, ids, flags)
        if rnd % 2:
            q.cancel(ids[::7])
        if rnd == 2:
            q.drain_launch("identity", peek=True, full_pickle=True)
            check(q.fetch(callbacks=True), key, m)
        if rnd == 3:
            for _ in range(3):
                q.drain_launch("identity", max_tasks=40, wait=False, full_pickle=True)
            check(q.fetch(callbacks=True), key, m)
        while q.depth():
            r = q.drain("identity", full_pickle=True, callbacks=True)
            check(r, key, m)
    q.close()


def test_enospc_then_a_fetch_that_fits():
    q = queue()
    q.set_callback_policy(b"k")
    q.set_callback_runners(endpoint=True)
    bodies = endpoint_bodies()
    ids = ids_for(len(bodies), 30)
    push(q, bodies, ids, [L.TF_HTTP_BODY] * len(bodies))
    q.drain_launch("identity", endpoint=True)
    st = q.stats()
    with pytest.raises(L.B9Error) as e:
        q.fetch(cap_bytes=int(st.last_drain_out_bytes) - 1, callbacks=True)
    assert e.value.code == L.B9_ENOSPC
    assert q.depth() == len(bodies)
    res = q.fetch(callbacks=True)
    check(res, b"k", {ids[i].tobytes(): ("ep", b) for i, b in enumerate(bodies)})
    assert q.depth() == 0
    q.close()


def test_runners_zero_unchanged_and_unknown_bits():
    q = queue()
    assert q._lib.b9_set_callback_runners(q._ctx, 4) == L.B9_EINVAL
    assert q._lib.b9_set_callback_runners(q._ctx, 0x100) == L.B9_EINVAL
    q.set_callback_policy(b"k")
    q.set_callback_runners()
    blobs = [frame_one("a"), frame_one([1, 2])]
    push(q, blobs, ids_for(2, 40), [L.TF_PICKLE] * 2)
    res = q.drain("identity", full_pickle=True, callbacks=True)
    assert list(res.cb_kind) == [cb.CB_HOST] * 2 and res.cb_body_len is None
    push(q, [b'{"args": ["x"]}'], ids_for(1, 41), [L.TF_HTTP_BODY])
    q.drain_launch("identity", endpoint=True)
    with pytest.raises(L.B9Error) as e:
        q.fetch(callbacks=True)
    assert e.value.code == L.B9_EINVAL
    q.close()


def test_baseline_function():
    """configs[4]'s 25 k documents pickled as `.map()` sends them, json_sum: every record against the oracle."""
    q = DeviceQueue(ring_bytes=1 << 30, ring_tasks=1 << 21, max_drain_tasks=1 << 21, max_result_bytes=1 << 30)
    q.set_callback_policy(b"key")
    q.set_callback_runners(function=True)
    b = synth.function_docs_batch(25_000)
    q.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, L.TF_PICKLE, np.uint8))
    res = q.drain("json_sum", callbacks=True, full_pickle=True)
    assert res.n == b.n
    raw = b.payload.tobytes()
    m = {b.task_ids[i].tobytes(): ("fn", raw[int(b.offsets[i]):int(b.offsets[i + 1])]) for i in range(b.n)}
    assert check(res, b"key", m) == {cb.CB_POST}
    q.close()


def test_baseline_endpoint():
    """configs[1]'s 1 Mi strings (1 % of them drawn from the adversarial pool: escapes, non-ASCII, astral characters) as
    HTTP bodies, identity: every record's kind, D and digest. D = json.dumps(json.loads(E)), which is T(E) for a
    JSONResponse body."""
    q = DeviceQueue(ring_bytes=1 << 30, ring_tasks=1 << 21, max_drain_tasks=1 << 21, max_result_bytes=1 << 30)
    q.set_callback_policy(b"key")
    q.set_callback_runners(endpoint=True)
    b = synth.strings_batch(1 << 20, 256)
    q.push_batch(b.task_ids, b.payload, b.offsets, flags=np.full(b.n, L.TF_HTTP_BODY, np.uint8))
    res = q.drain("identity", callbacks=True, endpoint=True)
    assert res.n == b.n and (res.cb_kind == cb.CB_POST).all() and (res.status == L.ST_COMPLETE).all()
    pl = res.payload.tobytes()
    lens = set()
    non_ascii = 0
    for i in range(res.n):
        o, n = int(res.offsets[i]), int(res.lengths[i])
        d = json.dumps(json.loads(pl[o:o + n])).encode()
        bo, bn = int(res.cb_body_off[i]), int(res.cb_body_len[i])
        assert pl[bo:bo + bn] == d, i
        non_ascii += bn != n
        lens.add(bn)
        body = cb0.BODY_PREFIX + d + b"}"
        assert res.cb_digest[i].tobytes() == hmac.new(b"key", cb0.sign_message(body, res.cb_timestamp), hashlib.sha256).digest(), i
    assert non_ascii > 1000 and len(lens) > 100                    # (the escape paths and mixed D lengths in a warp ran)
    q.close()


def test_enospc_function_runner_and_device_overflow():
    """B9_ENOSPC consumes nothing: the caller's cap_bytes below records + D for the function runner, and a staging
    (max_result_bytes) that holds the records but not their D bytes, for both runners."""
    key = b"k"
    blobs = [frame_one("é" * 100 + str(i)) for i in range(100)]
    q = queue()
    q.set_callback_policy(key)
    q.set_callback_runners(function=True)
    ids = ids_for(len(blobs), 50)
    push(q, blobs, ids, [L.TF_PICKLE] * len(blobs))
    q.drain_launch("identity", full_pickle=True)
    need = int(q.stats().last_drain_out_bytes)
    assert need > 100 * 600                                          # (the D bytes are counted)
    with pytest.raises(L.B9Error) as e:
        q.fetch(cap_bytes=need - 1, callbacks=True)
    assert e.value.code == L.B9_ENOSPC and q.depth() == len(blobs)
    res = q.fetch(callbacks=True)
    check(res, key, {ids[i].tobytes(): ("fn", b) for i, b in enumerate(blobs)})
    assert q.depth() == 0
    q.close()
    bodies = [b'{"args": ["' + ("é" * 100 + str(i)).encode() + b'"]}' for i in range(100)]
    for runner, payloads, flag, kw in (("function", blobs, L.TF_PICKLE, dict(full_pickle=True)),
                                       ("endpoint", bodies, L.TF_HTTP_BODY, dict(endpoint=True))):
        q = queue(max_result_bytes=1 << 16)                          # records ~ 22 KB, their D ~ 60 KB more
        q.set_callback_policy(key)
        push(q, payloads, ids_for(100, 60), [flag] * 100)
        q.drain_launch("identity", **kw)                             # without the runner's bit the records fit
        q.fetch(callbacks=runner == "function")
        push(q, payloads, ids_for(100, 61), [flag] * 100)
        q.set_callback_runners(**{runner: True})
        with pytest.raises(L.B9Error) as e:
            q.drain_launch("identity", **kw)
        assert e.value.code == L.B9_ENOSPC and q.depth() == 100, runner
        q.close()


def test_old_fetch_refuses_a_runner_launch():
    """b9_drain_fetch_callbacks does not return D, so it refuses a launch whose digests sign D; nothing is consumed."""
    q = queue()
    q.set_callback_policy(b"k")
    q.set_callback_runners(endpoint=True)
    bodies = [b'{"args": ["\\u00e9"]}', b'{"args": [[1, 2]]}']
    ids = ids_for(2, 70)
    push(q, bodies, ids, [L.TF_HTTP_BODY] * 2)
    q.drain_launch("identity", endpoint=True)
    runners, q._cb_runners = q._cb_runners, 0                        # (the binding would pick the new fetch)
    with pytest.raises(L.B9Error) as e:
        q.fetch(callbacks=True)
    assert e.value.code == L.B9_EINVAL and q.depth() == 2
    q._cb_runners = runners
    res = q.fetch(callbacks=True)
    check(res, b"k", {ids[i].tobytes(): ("ep", b) for i, b in enumerate(bodies)})
    q.close()


def test_sdk_mirrors():
    """Function(callback_url=...) and Endpoint(callback_url=...): each input's (url, body, headers) is the runner's, and
    what the calls return is unchanged."""
    from beta9_b200.endpoint import Endpoint
    from beta9_b200.function import Function
    key = b"sdk-key"
    f = Function(gpu_handler="identity", full_pickle=True, callback_url="http://stub", signing_key=key, queue=queue())(lambda x: x)
    values = ["a", [1, 2.5, None], {"k": "é"}, b"x", float("nan")]
    got = list(f.map([(v,) for v in values]))                      # (.map spreads a tuple as the arguments)
    assert got[:4] == values[:4] and got[4] != got[4]
    assert f.callbacks[3] is None and f.callbacks[4] is None
    for x, c in zip(values[:3], f.callbacks[:3]):
        url, body, headers = c
        assert url == "http://stub" and body == cb0.BODY_PREFIX + json.dumps(x).encode() + b"}"
        assert headers["X-Task-Status"] == "COMPLETE"
        assert headers["X-Task-Signature"] == cb0.sign_payload(body, key, int(headers["X-Task-Timestamp"]))[0]
    assert f.remote("s", callback_url="http://own") == "s"
    assert f.callbacks[0][0] == "http://own"
    e = Endpoint(gpu_handler="identity", callback_url="http://stub", signing_key=key, queue=queue())(lambda x: x)
    out = e.requests([b'{"args": ["\\u00e9"]}', b'not json', b'{"args": [[1, {"a": 2}]]}'])
    assert out[0] == (200, '"é"'.encode()) and out[1][0] == 400
    assert e.callbacks[1] is None
    assert e.callbacks[0][1] == b'{"data": "\\u00e9"}' and e.callbacks[2][1] == b'{"data": [1, {"a": 2}]}'
