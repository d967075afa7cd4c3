"""GPU: b9_wire_encode_full -- TaskMessage.Encode for floats, unsorted / duplicate keys and HTTP bodies.

* strict vs full: wherever b9_wire_encode answers, b9_wire_encode_full writes the same bytes (configs[1]-[3] shapes, every
  golden group);
* against the oracle: the golden wires and the Python oracle's records (loop.run_task_loop(keep_wire=True)) on the
  json_batch / json_float_batch / values_batch workloads, the float64 edge payloads and HTTP bodies; every decline is a
  documented one (tests/test_wire_full_on_host.py's decline_reasons), counted;
* round trip: every record pushed back with B9_TF_TASK_MSG drains, for every handler, exactly like its payload;
* edges: a wrapping 4 Ki-slot ring, max_result_bytes overflow, and drains after the call."""
import base64

import numpy as np
import pytest

from beta9_b200 import synth
from beta9_b200._lib import B9_ENOSPC, TF_HTTP_BODY, TF_TASK_MSG, B9Error
from oracle import coracle
from oracle.pyoracle import loop
from tests import golden_util as G
from tests.f64_corpus import sum_edge_payloads, value_edge_payloads
from tests.test_oracle_c_vs_py import HANDCRAFTED
from tests.test_wire_full_on_host import decline_reasons

pytestmark = pytest.mark.gpu
NOW = coracle.DEFAULT_NOW_NS
TTL = 7200
WS, STUB = coracle.DEFAULT_WS, coracle.DEFAULT_STUB
HANDLERS = ["identity", "crc32", "vadd_f32", "json_sum"]
KW_MERGED = b'{"kwargs": {"a": 1}, "kwargs": {}, "args": ["x"]}'


@pytest.fixture(scope="module")
def dq():
    from beta9_b200.device_queue import DeviceQueue
    q = DeviceQueue(ring_bytes=1 << 30, ring_tasks=1 << 20, max_drain_tasks=1 << 20, max_result_bytes=2 << 30)
    yield q
    q.close()


def push_with_meta(q, b, flags=None):
    n = b.n
    q.push_batch(b.task_ids, b.payload, b.offsets, timestamp_unix=np.full(n, NOW // 10**9, np.int64),
                 expires_unix_ns=np.full(n, NOW + TTL * 10**9, np.int64), flags=flags)


def encode(q, b, flags=None, strict=True):
    """(b9_wire_encode, b9_wire_encode_full) of batch b; the queue is empty again afterwards"""
    assert q.depth() == 0
    push_with_meta(q, b, flags)
    s = q.wire_encode(WS, STUB, ttl=TTL) if strict else None
    f = q.wire_encode(WS, STUB, ttl=TTL, full=True)
    assert q.depth() == b.n                             # peeks: nothing consumed
    q.drain("identity", max_tasks=b.n)
    assert q.depth() == 0 and f.n == b.n and np.array_equal(f.task_ids, b.task_ids)
    return s, f


def gather(r, idx) -> bytes:
    """the record bytes of r at the indices idx, concatenated"""
    return b"".join(r.payload[int(r.offsets[i]):int(r.offsets[i]) + int(r.lengths[i])].tobytes() for i in idx)


def assert_full_extends_strict(s, f, where=""):
    assert s.n == f.n and np.array_equal(s.task_ids, f.task_ids), where
    ok = np.flatnonzero(s.status == 0)
    assert (f.status[ok] == 0).all(), where
    assert (f.status[s.status == 3] == 3).all(), where
    assert np.array_equal(s.lengths[ok], f.lengths[ok]), where
    for lo in range(0, ok.size, 50_000):
        part = ok[lo:lo + 50_000]
        assert gather(s, part) == gather(f, part), where
    return ok.size


def check_against(f, payloads, want, http=False, where=""):
    """full records against the oracle's; returns the number of declines (each with a documented reason)"""
    declined = 0
    for i, (p, w) in enumerate(zip(payloads, want)):
        if w.status == loop.REJECTED:
            assert f.status[i] == 3 and not f.has_result[i], (where, p[:120])
        elif f.status[i] == 4:
            assert decline_reasons(p, http), (where, p[:200])
            declined += 1
        else:
            assert f.status[i] == 0 and f.result(i) == w.wire, (where, p[:200], f.result(i), w.wire)
    return declined


def oracle_records(payloads, b, http=False):
    ids = [bytes(b.task_ids[i]) for i in range(b.n)]
    return loop.run_task_loop(payloads, ids, "identity", keep_wire=True, now_unix_ns=NOW, http_body=http)


# ---------------------------------------------------------------------------------------------- strict vs full
def test_strict_and_full_agree_where_strict_answers(dq):
    for name, b in (("configs1_strings", synth.strings_batch(1_000_000, 256, adversarial_frac=0.01)),
                    ("crc", synth.crc_batch(200_000)), ("vadd", synth.vadd_batch(200_000))):
        s, f = encode(dq, b)
        assert_full_extends_strict(s, f, name)
        assert int((f.status == 4).sum()) == 0, name


def test_golden_groups(dq):
    g = G.load()
    declined = []
    for name, cases in g["groups"].items():
        b = G.group_batch(cases)
        assert dq.depth() == 0
        push_with_meta(dq, b)
        s = dq.wire_encode(g["workspace"], g["stub"], ttl=TTL)
        f = dq.wire_encode(g["workspace"], g["stub"], ttl=TTL, full=True)
        dq.drain("identity", max_tasks=b.n)
        assert_full_extends_strict(s, f, name)
        for i, c in enumerate(cases):
            want = base64.b64decode(c["wire"]) if c["wire"] else None
            p = base64.b64decode(c["payload"])
            if f.status[i] == 4:
                declined.append((name, p))
                continue
            if want is None:
                assert f.status[i] == 3, (name, i, p)
            else:
                assert f.status[i] == 0 and f.result(i) == want, (name, i, p, f.result(i), want)
        if name == "handcrafted":
            newly = [p for i, p in enumerate(base64.b64decode(c["payload"]) for c in cases) if s.status[i] == 4 and f.status[i] == 0]
            for p in (b'{"args": [1.0]}', b'{"args": [1e3]}', b'{"args": [1.5]}', b'{"args": [9007199254740992]}',
                      b'{"args": [9007199254740994]}', b'{"args": [{"b": 1, "a": 2, "b": 3}]}', b'{"args": [{"values": [1], "values": [5, 6]}]}',
                      b'{"args": [[1, "a", null, true, {"b": [], "a": "<"}]]}', b'{"args": [{"values": [1.5]}]}'):
                assert p in newly, p
    assert declined == [("handcrafted", KW_MERGED)], declined


# ---------------------------------------------------------------------------------------------- against the oracle
def test_json_batch_all_answered(dq):
    """configs[4]'s shape, {"id", "values", "pad"}: every record answered and equal to the C oracle's (which is the Python
    oracle's for this shape; the Python oracle itself checks the first 5000)"""
    b = synth.json_batch(100_000)
    _, f = encode(dq, b, strict=False)
    assert int((f.status != 0).sum()) == 0
    o = coracle.run_batch(b.task_ids, b.payload, b.offsets, "identity", keep_wire=True, nthreads=8)
    assert (o.status == 0).all()
    for lo in range(0, b.n, 20_000):
        idx = range(lo, min(b.n, lo + 20_000))
        assert gather(f, idx) == b"".join(o.wire_msg(i) for i in idx), lo
    head = synth.from_payloads([b.task(i) for i in range(5000)])
    head.task_ids = b.task_ids[:5000].copy()
    want = oracle_records(head.tasks(), head)
    assert all(f.result(i) == want[i].wire for i in range(5000))


@pytest.mark.parametrize("kind", ["json_float_batch", "values_batch", "f64_edges"])
def test_float_and_value_workloads(dq, kind):
    if kind == "json_float_batch":
        b = synth.json_float_batch(5_000)
    elif kind == "values_batch":
        b = synth.values_batch(20_000)
    else:
        b = synth.from_payloads([p for p, _ in sum_edge_payloads()] + [p for p, _ in value_edge_payloads()])
    payloads = b.tasks()
    _, f = encode(dq, b, strict=False)
    declined = check_against(f, payloads, oracle_records(payloads, b), where=kind)
    print(f"\n{kind}: {b.n} tasks, {declined} declined")
    if kind == "f64_edges":                             # (the corpus seeks out the limits: 17 levels, 65 members, 20+ digits)
        assert declined <= b.n // 10, declined
    else:
        assert declined == 0


def test_http_bodies(dq):
    bodies = list(HANDCRAFTED) + [b'{"x": 1.5, "args": [1], "b": {"z": 1, "a": 2}}', b'{"args": "s", "k": 1e2}', b'{"kwargs": 5, "y": [1.0]}',
                                  b'{"args": [1], "args": "s"}', b'{"args": "s", "args": [1], "zz": -0.0}', b" null ", b"\n",
                                  b'{"kwargs": {"b": 1, "a": 2}, "kwargs": [3]}', b'{"a": 1, "\\u0061": 2, "args": [], "\\u0061rgs": 7}']
    b = synth.from_payloads(bodies)
    flags = np.full(b.n, TF_HTTP_BODY, np.uint8)
    _, f = encode(dq, b, flags, strict=False)
    declined = check_against(f, bodies, oracle_records(bodies, b, http=True), http=True, where="http")
    assert declined == 0


# ---------------------------------------------------------------------------------------------- round trip
def test_records_drain_like_their_payloads(dq):
    parts = [synth.json_batch(20_000, seed=3), synth.json_float_batch(5_000, seed=4), synth.values_batch(20_000, seed=5),
             synth.strings_batch(20_000, 128, adversarial_frac=0.2, seed=6), synth.vadd_batch(5_000, seed=7),
             synth.from_payloads(list(HANDCRAFTED)), synth.from_payloads(list(HANDCRAFTED))]
    b = synth.concat(parts)
    flags = np.zeros(b.n, np.uint8)
    flags[b.n - len(HANDCRAFTED):] = TF_HTTP_BODY          # the last copy of HANDCRAFTED as HTTP bodies
    _, f = encode(dq, b, flags, strict=False)
    enc = np.flatnonzero(f.status == 0)
    assert enc.size >= 0.97 * b.n
    recs = synth.from_payloads([f.result(int(i)) for i in enc])
    recs.task_ids = b.task_ids[enc].copy()
    for handler in HANDLERS:
        dq.push_batch(b.task_ids, b.payload, b.offsets, flags=flags)
        want = dq.drain(handler, max_tasks=b.n)
        dq.push_batch(recs.task_ids, recs.payload, recs.offsets, flags=np.full(recs.n, TF_TASK_MSG, np.uint8))
        got = dq.drain(handler, max_tasks=recs.n)
        assert dq.depth() == 0 and got.n == enc.size and np.array_equal(got.task_ids, b.task_ids[enc])
        bad = np.flatnonzero((got.status == 4) & (want.status[enc] != 4))
        assert bad.size == 0, (handler, [recs.task(int(i))[:160] for i in bad[:3]])
        assert np.array_equal(got.status, want.status[enc]), handler
        assert np.array_equal(got.has_result, want.has_result[enc]) and np.array_equal(got.lengths, want.lengths[enc]), handler
        assert gather(got, range(got.n)) == gather(want, enc), handler


# ---------------------------------------------------------------------------------------------- edges
def _mixed(seed: int):
    vb = synth.values_batch(3_000, seed=seed)
    fb = synth.json_float_batch(1_000, seed=seed + 1)
    hb = synth.from_payloads(list(HANDCRAFTED) * 5)
    b = synth.concat([vb, fb, hb])
    flags = np.zeros(b.n, np.uint8)
    flags[vb.n + fb.n:] = TF_HTTP_BODY
    payloads = b.tasks()
    want = {}
    for lo, hi, http in ((0, vb.n + fb.n, False), (vb.n + fb.n, b.n, True)):
        sub = synth.from_payloads(payloads[lo:hi])
        sub.task_ids = b.task_ids[lo:hi].copy()
        for i, w in zip(range(lo, hi), oracle_records(payloads[lo:hi], sub, http)):
            want[b.task_ids[i].tobytes()] = (payloads[i], w, http)
    return b, flags, want


def test_wrapping_ring():
    from beta9_b200.device_queue import DeviceQueue
    b, flags, want = _mixed(101)
    rng = np.random.default_rng(102)
    checked = 0
    with DeviceQueue(ring_bytes=1 << 22, ring_tasks=1 << 12, max_drain_tasks=1 << 12, max_result_bytes=1 << 24) as q:
        lo = 0
        while lo < b.n or q.depth():
            while lo < b.n and q.depth() < 3000:
                hi = min(b.n, lo + int(rng.integers(1, 600)))
                sub = synth.from_payloads([b.task(i) for i in range(lo, hi)])
                sub.task_ids = b.task_ids[lo:hi].copy()
                try:
                    push_with_meta(q, sub, flags[lo:hi])
                except B9Error as e:
                    assert e.code == B9_ENOSPC
                    break
                lo = hi
            f = q.wire_encode(WS, STUB, ttl=TTL, full=True)
            assert f.n == q.depth()
            for i in range(f.n):
                p, w, http = want[f.task_ids[i].tobytes()]
                if w.status == loop.REJECTED:
                    assert f.status[i] == 3
                elif f.status[i] == 4:
                    assert decline_reasons(p, http), p[:160]
                else:
                    assert f.status[i] == 0 and f.result(i) == w.wire, p[:160]
                checked += 1
            q.drain("identity", max_tasks=int(rng.integers(1, 1500)))
    assert checked >= b.n


def test_overflow_leaves_the_queue_alone():
    from beta9_b200.device_queue import DeviceQueue
    b = synth.json_float_batch(2_000, seed=111)
    with DeviceQueue(ring_bytes=1 << 24, ring_tasks=1 << 12, max_drain_tasks=1 << 12, max_result_bytes=1 << 16) as q:
        push_with_meta(q, b)
        with pytest.raises(B9Error) as e:
            q.wire_encode(WS, STUB, ttl=TTL, full=True)
        assert e.value.code == B9_ENOSPC and q.depth() == b.n
        f = q.wire_encode(WS, STUB, ttl=TTL, full=True, max_tasks=8)            # a window that fits
        assert f.n == 8 and q.depth() == b.n and (f.status == 0).all()
        r = q.drain("identity", max_tasks=8)                                    # (the staging is sized for the overflow)
        assert r.n == 8 and q.depth() == b.n - 8 and np.array_equal(r.task_ids, b.task_ids[:8])


def test_drains_after_full_encode_equal_a_fresh_queue(dq):
    from beta9_b200.device_queue import DeviceQueue
    b, flags, _ = _mixed(121)
    with DeviceQueue(ring_bytes=1 << 26, ring_tasks=1 << 15, max_drain_tasks=1 << 15, max_result_bytes=1 << 26) as fresh:
        for handler in ("identity", "json_sum"):
            fresh.push_batch(b.task_ids, b.payload, b.offsets, flags=flags)
            want = fresh.drain(handler, max_tasks=b.n)
            # blocking drain after the call
            dq.push_batch(b.task_ids, b.payload, b.offsets, flags=flags)
            dq.wire_encode(WS, STUB, ttl=TTL, full=True)
            _same(dq.drain(handler, max_tasks=b.n), want, (handler, "blocking"))
            # a burst of async peek drains after the call, then the blocking one
            dq.push_batch(b.task_ids, b.payload, b.offsets, flags=flags)
            dq.wire_encode(WS, STUB, ttl=TTL, full=True)
            for _ in range(4):
                assert dq.drain_launch(handler, b.n, peek=True, wait=False) == b.n
            _same(dq.fetch(), want, (handler, "burst"))
            _same(dq.drain(handler, max_tasks=b.n), want, (handler, "after burst"))
            assert dq.depth() == 0


def _same(a, b, where):
    assert a.n == b.n and np.array_equal(a.task_ids, b.task_ids), where
    assert np.array_equal(a.status, b.status) and np.array_equal(a.has_result, b.has_result), where
    assert np.array_equal(a.lengths, b.lengths) and np.array_equal(a.fifo_payload(), b.fifo_payload()), where
