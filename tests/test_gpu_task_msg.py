"""GPU: TaskMessage records pushed with B9_TF_TASK_MSG, drained by every handler.

* the golden wire records against the reference runner's own answers (tests/golden/ref_runner_golden.json);
* round trips at the configurations' sizes: draining the oracle's records of a batch gives, task by task, exactly
  what draining the batch's payloads gives (status, has_result, bytes); configs[1]'s records are all answered;
* b9_wire_encode -> fetch -> push the records with the flag -> drain, against draining the payloads;
* records mixed with SDK payloads, HTTP bodies, pickles and cancelled tasks; a small wrapping ring with partial drains;
  a queue with a 1 KiB stage buffer (records unstaged); the CPU test's mutants, never answered wrong."""
import base64
import json
import os

import numpy as np
import pytest

from beta9_b200 import synth
from beta9_b200._lib import TF_CANCELLED, TF_HTTP_BODY, TF_PICKLE, TF_TASK_MSG, B9Error
from oracle import coracle
from oracle.pyoracle import loop
from tests.task_msg_oracle import NOT_RUN, run_records

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
HANDLERS = ["identity", "crc32", "vadd_f32", "json_sum"]
CODE = {"COMPLETE": 0, "ERROR": 1, "RETRY": 2, "REJECTED": 3, NOT_RUN: 4}


@pytest.fixture(scope="module")
def dq():
    from beta9_b200.device_queue import DeviceQueue
    q = DeviceQueue(ring_bytes=1 << 32, ring_tasks=1 << 21, max_drain_tasks=1 << 21, max_result_bytes=1 << 30)   # configs[2]'s records: 1.3 GB
    yield q
    q.close()


@pytest.fixture(scope="module")
def dq_small_stage():
    from beta9_b200.device_queue import DeviceQueue
    old = os.environ.get("B9_STAGE_BYTES")
    os.environ["B9_STAGE_BYTES"] = "1024"
    try:
        q = DeviceQueue(ring_bytes=1 << 28, ring_tasks=1 << 18, max_drain_tasks=1 << 18, max_result_bytes=1 << 28)
    finally:
        if old is None:
            del os.environ["B9_STAGE_BYTES"]
        else:
            os.environ["B9_STAGE_BYTES"] = old
    yield q
    q.close()


def pack(ids: np.ndarray, blobs) -> synth.Batch:
    lens = np.array([len(b) for b in blobs], np.uint64)
    off = np.zeros(len(blobs) + 1, np.uint64)
    np.cumsum(lens, out=off[1:])
    pl = np.frombuffer(b"".join(blobs), np.uint8) if blobs else np.empty(0, np.uint8)
    return synth.Batch(np.ascontiguousarray(ids, np.uint8).reshape(-1, 16), pl, off, "records")


def drain_all(q, batch: synth.Batch, handler: str, flags=None):
    assert q.depth() == 0
    q.push_batch(batch.task_ids, batch.payload, batch.offsets, flags=flags)
    r = q.drain(handler, max_tasks=batch.n)
    assert q.depth() == 0 and r.n_popped == batch.n
    return r


def same_records(a, b, where=""):
    """two drains of the same tasks: identical ids, status, has_result, lengths and bytes, record by record"""
    assert a.n == b.n, where
    assert np.array_equal(a.task_ids, b.task_ids), where
    bad = np.flatnonzero((a.status != b.status) | (a.has_result != b.has_result) | (a.lengths != b.lengths))
    assert bad.size == 0, (where, bad[:5], a.status[bad[:5]], b.status[bad[:5]])
    assert np.array_equal(a.fifo_payload(), b.fifo_payload()), where


def c_oracle_records(batch: synth.Batch, handler: str):
    o = coracle.run_batch(batch.task_ids, batch.payload, batch.offsets, handler, nthreads=os.cpu_count() or 1, keep_wire=True)
    return [o.wire_msg(i) for i in range(batch.n)]


def record_flags(n: int) -> np.ndarray:
    return np.full(n, TF_TASK_MSG, np.uint8)


# ---------------------------------------------------------------------------------------------- 4. goldens
@pytest.mark.parametrize("handler", HANDLERS)
def test_golden_records_against_the_reference_runner(dq, handler):
    hot = json.load(open(os.path.join(HERE, "golden", "hot_path_golden.json")))
    ref = json.load(open(os.path.join(HERE, "golden", "ref_runner_golden.json")))
    cases = [(g, i, c) for g, cs in hot["groups"].items() for i, c in enumerate(cs) if c["wire"] is not None]
    ids = np.stack([np.frombuffer(bytes.fromhex(c["task_id"]), np.uint8) for _, _, c in cases])
    recs = pack(ids, [base64.b64decode(c["wire"]) for _, _, c in cases])
    pays = pack(ids, [base64.b64decode(c["payload"]) for _, _, c in cases])
    r = drain_all(dq, recs, handler, record_flags(recs.n))
    p = drain_all(dq, pays, handler)
    assert r.n == len(cases) and np.array_equal(r.task_ids, ids)
    for k, (g, i, _) in enumerate(cases):
        r_status, r_result, _ = ref["groups"][g][str(i)][handler]
        if int(r.status[k]) == 4:
            assert int(p.status[k]) == 4, (g, i, "a Go-written record declined whose payload is answered")
            continue
        assert int(r.status[k]) == CODE[r_status], (g, i)
        assert r.result(k) == (None if r_result is None else base64.b64decode(r_result)), (g, i)


# ---------------------------------------------------------------------------------------------- 5. round trips at size
ROUND_TRIPS = {
    "configs1_identity": (lambda: synth.strings_batch(1_000_000, 256), "identity"),
    "configs2_crc32": (lambda: synth.crc_batch(1_000_000), "crc32"),
    "configs3_vadd_f32": (lambda: synth.vadd_batch(1_250_000), "vadd_f32"),
    "configs4_json_sum": (lambda: synth.json_batch(25_000), "json_sum"),
}


@pytest.mark.parametrize("name", list(ROUND_TRIPS))
def test_round_trip_at_size(dq, name):
    make, handler = ROUND_TRIPS[name]
    b = make()
    recs = pack(b.task_ids, c_oracle_records(b, handler))
    want = drain_all(dq, b, handler)
    got = drain_all(dq, recs, handler, record_flags(b.n))
    same_records(got, want, name)
    if name == "configs1_identity":
        assert int((got.status == 4).sum()) == 0


@pytest.mark.parametrize("kind", ["values", "floats"])
def test_round_trip_float_and_container_values(dq, kind):
    b = synth.values_batch(20_000, seed=51) if kind == "values" else synth.json_float_batch(5_000, seed=52)
    ids = [bytes(b.task_ids[i]) for i in range(b.n)]
    live = loop.run_task_loop(b.tasks(), ids, "identity", keep_wire=True)
    assert all(w.wire is not None for w in live)
    recs = pack(b.task_ids, [w.wire for w in live])
    for handler in ("identity", "json_sum"):
        want = drain_all(dq, b, handler)
        got = drain_all(dq, recs, handler, record_flags(b.n))
        same_records(got, want, (kind, handler))


# ---------------------------------------------------------------------------------------------- 6. device encoder -> records
def test_wire_encode_records_drain_like_their_payloads(dq):
    parts = [synth.strings_batch(40_000, 256, seed=61), synth.json_batch(2_000, seed=62), synth.crc_batch(5_000, seed=63)]
    b = synth.concat(parts)
    dq.push_batch(b.task_ids, b.payload, b.offsets)
    w = dq.wire_encode("ws-b200", "7f1c2d3e-4a5b-4c6d-8e9f-0a1b2c3d4e5f")
    assert w.n == b.n and dq.depth() == b.n
    enc = np.flatnonzero(w.status == 0)
    assert enc.size > 0.9 * b.n
    for handler in ("identity", "crc32", "json_sum"):
        if dq.depth() == 0:
            dq.push_batch(b.task_ids, b.payload, b.offsets)
        want = dq.drain(handler, max_tasks=b.n)
        assert dq.depth() == 0
        recs = pack(b.task_ids[enc], [w.result(int(i)) for i in enc])
        got = drain_all(dq, recs, handler, record_flags(recs.n))
        assert np.array_equal(got.task_ids, b.task_ids[enc])
        assert np.array_equal(got.status, want.status[enc]) and np.array_equal(got.has_result, want.has_result[enc]), handler
        assert np.array_equal(got.lengths, want.lengths[enc]), handler
        for i in range(0, enc.size, 97):
            assert got.result(i) == want.result(int(enc[i])), (handler, i)
    # the encoder does not encode a record again
    rec1 = pack(b.task_ids[:4], [w.result(0), w.result(1), w.result(2), w.result(3)])
    dq.push_batch(rec1.task_ids, rec1.payload, rec1.offsets, flags=record_flags(4))
    w2 = dq.wire_encode("ws-b200", "stub")
    assert list(w2.status) == [4, 4, 4, 4]
    dq.drain("identity")


# ---------------------------------------------------------------------------------------------- 7. mixed and edge cases
def mixed_batch(seed: int):
    """records, SDK payloads, HTTP bodies, pickles and cancelled tasks interleaved; the flags and, per task, what it is"""
    from oracle.pyoracle import funcloop
    rng = np.random.default_rng(seed)
    s = synth.strings_batch(6_000, 200, adversarial_frac=0.05, seed=seed)
    v = synth.values_batch(1_500, seed=seed + 1)
    base = synth.concat([s, v])
    ids = [bytes(base.task_ids[i]) for i in range(base.n)]
    live = loop.run_task_loop(base.tasks(), ids, "identity", keep_wire=True)
    blobs, flags, kinds = [], [], []
    for i in range(base.n):
        k = int(rng.integers(0, 10))
        if k < 5:
            blobs.append(live[i].wire); flags.append(TF_TASK_MSG); kinds.append("record")
        elif k < 7:
            blobs.append(base.task(i)); flags.append(0); kinds.append("sdk")
        elif k == 7:
            blobs.append(base.task(i)); flags.append(TF_HTTP_BODY); kinds.append("http")
        elif k == 8:
            blobs.append(funcloop.frame_map_input("x" * int(rng.integers(0, 80)))); flags.append(TF_PICKLE); kinds.append("pickle")
        else:
            blobs.append(live[i].wire); flags.append(TF_TASK_MSG | TF_CANCELLED); kinds.append("cancelled")
    return pack(base.task_ids, blobs), np.array(flags, np.uint8), kinds


def expected_by_kind(q, batch, flags, kinds, handler):
    """every task's answer, from drains that each hold one kind of task"""
    want = {}
    for kind in ("record", "sdk", "http", "pickle"):
        idx = [i for i, k in enumerate(kinds) if k == kind]
        sub = pack(batch.task_ids[idx], [batch.task(i) for i in idx])
        r = drain_all(q, sub, handler, flags[idx])
        for j, i in enumerate(idx):
            want[i] = (int(r.status[j]), r.result(j))
    return want


@pytest.mark.parametrize("handler", ["identity", "crc32", "json_sum"])
def test_records_mixed_with_other_tasks(dq, handler):
    batch, flags, kinds = mixed_batch(71)
    want = expected_by_kind(dq, batch, flags, kinds, handler)
    r = drain_all(dq, batch, handler, flags)
    live = [i for i, k in enumerate(kinds) if k != "cancelled"]
    assert r.n == len(live) and np.array_equal(r.task_ids, batch.task_ids[live])
    for j, i in enumerate(live):
        assert (int(r.status[j]), r.result(j)) == want[i], (kinds[i], batch.task(i)[:120])
    # records answered per the record oracle
    rec_idx = [i for i, k in enumerate(kinds) if k == "record"]
    o = run_records([batch.task(i) for i in rec_idx], [bytes(batch.task_ids[i]) for i in rec_idx], handler)
    for i, w in zip(rec_idx, o):
        st, res = want[i]
        assert st == 4 or (st == CODE[w.status] and res == w.result), batch.task(i)[:120]
    if handler == "identity":
        assert all(want[i][0] != 4 for i in rec_idx)


def test_small_wrapping_ring_with_partial_drains():
    from beta9_b200.device_queue import DeviceQueue
    batch, flags, kinds = mixed_batch(81)
    with DeviceQueue(ring_bytes=1 << 21, ring_tasks=1 << 12, max_drain_tasks=1 << 12, max_result_bytes=1 << 22) as q, \
         DeviceQueue(ring_bytes=1 << 26, ring_tasks=1 << 15, max_drain_tasks=1 << 15, max_result_bytes=1 << 26) as ref_q:
        want = expected_by_kind(ref_q, batch, flags, kinds, "identity")
        rng = np.random.default_rng(82)
        got = {}
        lo = 0
        while lo < batch.n or q.depth():
            while lo < batch.n and q.depth() < 2500:
                hi = min(batch.n, lo + int(rng.integers(1, 700)))
                sub = pack(batch.task_ids[lo:hi], [batch.task(i) for i in range(lo, hi)])
                try:
                    q.push_batch(sub.task_ids, sub.payload, sub.offsets, flags=flags[lo:hi])
                except B9Error as e:
                    assert e.code == -28                       # B9_ENOSPC: the ring is full, drain first
                    break
                lo = hi
            r = q.drain("identity", max_tasks=int(rng.integers(1, 900)))
            for j in range(r.n):
                got[r.task_ids[j].tobytes()] = (int(r.status[j]), r.result(j))
        for i in range(batch.n):
            if kinds[i] != "cancelled":
                assert got[batch.task_ids[i].tobytes()] == want[i], (kinds[i], batch.task(i)[:120])


def test_unstaged_records_are_byte_identical(dq, dq_small_stage):
    b = synth.concat([synth.strings_batch(20_000, 256, seed=91), synth.values_batch(5_000, seed=92)])
    ids = [bytes(b.task_ids[i]) for i in range(b.n)]
    recs = pack(b.task_ids, [w.wire for w in loop.run_task_loop(b.tasks(), ids, "identity", keep_wire=True)])
    for handler in ("identity", "crc32", "json_sum"):
        same_records(drain_all(dq_small_stage, recs, handler, record_flags(b.n)), drain_all(dq, recs, handler, record_flags(b.n)), handler)


def test_mutants_are_never_answered_wrong(dq):
    from tests.test_task_msg_on_host import MUTANTS, TID
    rng = np.random.default_rng(101)
    seeds = [m for m, want in MUTANTS.values() if want == "answer"]
    alphabet = list(b'{}[],:" 0159e.-+Etrun\\lfa') + [0x00, 0x1F, 0x7F, 0xC3, 0xA9, 0xED, 0xA0, 0xFF]
    blobs = [m for m, _ in MUTANTS.values()]
    for _ in range(20_000):
        m = bytearray(seeds[int(rng.integers(0, len(seeds)))])
        pos = int(rng.integers(0, len(m)))
        op = int(rng.integers(0, 3))
        ch = int(rng.choice(alphabet))
        if op == 0: m[pos] = ch
        elif op == 1: del m[pos]
        else: m[pos:pos] = bytes([ch])
        blobs.append(bytes(m))
    ids = np.tile(np.frombuffer(TID, np.uint8), (len(blobs), 1))
    recs = pack(ids, blobs)
    for handler in HANDLERS:
        r = drain_all(dq, recs, handler, record_flags(recs.n))
        o = run_records(blobs, [TID] * len(blobs), handler)
        answered = 0
        for j, w in enumerate(o):
            if int(r.status[j]) == 4:
                continue
            answered += 1
            assert w.status != NOT_RUN and int(r.status[j]) == CODE[w.status] and r.result(j) == w.result, (handler, blobs[j][:160])
        for j, (name, (_, want)) in enumerate(MUTANTS.items()):
            if want == "decline":
                assert int(r.status[j]) == 4, (handler, name)
        assert answered > 2_000, answered
