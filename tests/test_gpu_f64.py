"""GPU: the device build of the float64 codec and of the two handlers built on it, at the scale of the host tests.

- identity over `{"args": [L], "kwargs": {}}` and json_sum over `{"args": [{"values": [L]}], "kwargs": {}}` for every
  literal of f64_corpus._literals(), against the one-number restatements (pinned against the task loop on a CPU by
  test_f64_edges_on_host.py);
- json_sum over repr(x) and "%.17g" % x of B9_F64_PATTERNS random finite doubles (default 10M, in chunks of 1M) and of
  f64_corpus._powers();
- the json_sum and identity edge corpora against the oracle's task loop;
- the literals and the edge corpora again on a queue made with B9_STAGE_BYTES=1024, whose records must be
  byte-identical: there identity's value tasks are walked from global memory by the kernel's tail and json_sum's
  documents are parsed in place instead of from the warp's stage buffer;
- the edge corpora mixed into values_batch / json_float_batch tasks, pushed into a small ring in many small batches
  with partial drains, so that tiles span pushes and the ring wraps.

A task may be declined (B9_ST_UNSUPPORTED) only where the host tests allow it: a literal of more than 19 significant
digits, an int outside a C long, nesting deeper than 16 levels, an object of more than 64 members."""
import dataclasses
import os
from decimal import Decimal

import numpy as np
import pytest

from beta9_b200 import synth
from oracle.pyoracle import loop
from tests.f64_corpus import (C_LONG_MAX, C_LONG_MIN, _literals, _patterns, _powers, identity_of_literal, json_sum_of_literal,
                              literal_may_decline, sum_edge_payloads, value_edge_payloads)

pytestmark = pytest.mark.gpu
CODE = {"COMPLETE": 0, "ERROR": 1, "RETRY": 2, "REJECTED": 3}
N_PATTERNS = int(os.environ.get("B9_F64_PATTERNS", 10_000_000))
PUSH = 1 << 20                                                   # tasks per push


@dataclasses.dataclass
class Records:
    status: np.ndarray        # uint8 [n]
    has: np.ndarray           # bool [n]
    lengths: np.ndarray       # int64 [n], 0 where there is no result
    blob: bytes               # the result bytes in task order

    def result(self, i: int):
        if not self.has[i]:
            return None
        o = int(self.lengths[:i].sum())
        return self.blob[o:o + int(self.lengths[i])]


def _queue():
    from beta9_b200.device_queue import DeviceQueue
    return DeviceQueue(ring_bytes=1 << 30, ring_tasks=1 << 21, max_drain_tasks=1 << 21, max_result_bytes=1 << 30)


@pytest.fixture(scope="module")
def queues():
    """The default queue, and one whose warps have a 1 KiB stage buffer (B9_STAGE_BYTES is read when a queue is made)."""
    q = _queue()
    old = os.environ.get("B9_STAGE_BYTES")
    os.environ["B9_STAGE_BYTES"] = "1024"
    try:
        small = _queue()
    finally:
        if old is None:
            del os.environ["B9_STAGE_BYTES"]
        else:
            os.environ["B9_STAGE_BYTES"] = old
    yield q, small
    small.close()
    q.close()


def drain_all(q, payloads, handler) -> Records:
    st, has, ln, blobs = [], [], [], []
    for lo in range(0, len(payloads), PUSH):
        b = synth.from_payloads(payloads[lo:lo + PUSH], seed=lo)
        assert q.depth() == 0
        q.push_batch(b.task_ids, b.payload, b.offsets)
        r = q.drain(handler, max_tasks=b.n)
        assert r.n_popped == b.n and r.n == b.n and q.depth() == 0
        assert np.array_equal(r.task_ids, b.task_ids)
        h = r.has_result != 0
        lens = np.where(h, r.lengths, 0).astype(np.uint32)
        st.append(r.status.copy())
        has.append(h)
        ln.append(lens.astype(np.int64))
        blobs.append(dataclasses.replace(r, lengths=lens).fifo_payload().tobytes())
    return Records(np.concatenate(st), np.concatenate(has), np.concatenate(ln), b"".join(blobs))


def check(rec: Records, payloads, want_status, want_res, may_decline):
    """Every record against the expected (status, bytes); a decline only where `may_decline` allows it."""
    n = len(payloads)
    want_status = np.asarray(want_status, np.uint8)
    may_decline = np.asarray(may_decline, bool)
    assert rec.status.shape == (n,) and want_status.shape == (n,) and may_decline.shape == (n,) and len(want_res) == n
    dec = rec.status == 4
    bad = np.flatnonzero(dec & ~may_decline)
    assert bad.size == 0, ("declined", bad.size, payloads[bad[0]][:300])
    assert not (dec & rec.has).any()
    keep = ~dec
    want_has = np.array([w is not None for w in want_res], bool)
    want_len = np.array([len(w) if w is not None else 0 for w in want_res], np.int64)
    bad = np.flatnonzero(keep & ((rec.status != want_status) | (rec.has != want_has) | (rec.lengths != want_len)))
    if bad.size:
        i = int(bad[0])
        raise AssertionError((bad.size, payloads[i][:300], int(rec.status[i]), rec.result(i), int(want_status[i]), want_res[i]))
    want_blob = b"".join(w for w, k in zip(want_res, keep.tolist()) if k and w is not None)
    if rec.blob != want_blob:
        ends = np.cumsum(rec.lengths)
        first = next(k for k in range(min(len(rec.blob), len(want_blob)) + 1) if rec.blob[k:k + 1] != want_blob[k:k + 1])
        i = int(np.searchsorted(ends, first, side="right"))
        raise AssertionError((payloads[i][:300], rec.result(i), want_res[i]))
    return int(dec.sum())


def assert_same_records(a: Records, b: Records, payloads):
    bad = np.flatnonzero((a.status != b.status) | (a.has != b.has) | (a.lengths != b.lengths))
    assert bad.size == 0, (bad.size, payloads[int(bad[0])][:300], int(a.status[bad[0]]), int(b.status[bad[0]]))
    assert a.blob == b.blob


def _literal_payloads(wrap_open: bytes, wrap_close: bytes):
    lits = _literals()
    assert len(lits) >= 1_050_000
    return lits, [wrap_open + s.encode() + wrap_close for s in lits]


def test_identity_over_every_literal(queues):
    lits, payloads = _literal_payloads(b'{"args": [', b'], "kwargs": {}}')
    want = [identity_of_literal(s) for s in lits]
    rec = drain_all(queues[0], payloads, "identity")
    declined = check(rec, payloads, [w[0] for w in want], [w[1] for w in want], [literal_may_decline(s) for s in lits])
    assert_same_records(rec, drain_all(queues[1], payloads, "identity"), payloads)
    print(f"\nidentity: {len(lits)} literals, {declined} declined (> 19 significant digits)")


def test_json_sum_over_every_literal(queues):
    lits, payloads = _literal_payloads(b'{"args": [{"values": [', b']}], "kwargs": {}}')
    want = [json_sum_of_literal(s) for s in lits]
    rec = drain_all(queues[0], payloads, "json_sum")
    declined = check(rec, payloads, [w[0] for w in want], [w[1] for w in want], [w[2] for w in want])
    assert_same_records(rec, drain_all(queues[1], payloads, "json_sum"), payloads)
    print(f"\njson_sum: {len(lits)} literals, {declined} declined (> 19 significant digits or beyond a C long)")


def _expect_doubles(bits: np.ndarray):
    """json_sum of one double x written as repr(x) or "%.17g" % x (both parse back to x exactly): f64_corpus's
    json_sum_of_literal, with the int test vectorized. Returns the repr texts, the results and where a decline is allowed
    (an int beyond a C long); the status is always COMPLETE."""
    xs = bits.view(np.float64)
    integral = (xs == np.trunc(xs)) & (np.abs(xs) < 1e21)
    reprs = list(map(repr, xs.tolist()))
    res = [r.encode() for r in reprs]
    decline = np.zeros(xs.size, bool)
    for i in np.flatnonzero(integral).tolist():
        v = int(Decimal(reprs[i]))
        res[i] = str(v).encode() if v else None
        decline[i] = not C_LONG_MIN <= v <= C_LONG_MAX
    return reprs, res, decline


def test_json_sum_over_random_doubles(queues):
    done = 0
    chunks = [_patterns(1_000_000, 3000 + k) for k in range(max(1, N_PATTERNS // 1_000_000))] + [_powers()]
    for bits in chunks:
        reprs, res, decline = _expect_doubles(bits)
        texts = reprs + ["%.17g" % x for x in bits.view(np.float64).tolist()]
        payloads = [b'{"args": [{"values": [' + t.encode() + b']}], "kwargs": {}}' for t in texts]
        rec = drain_all(queues[0], payloads, "json_sum")
        check(rec, payloads, np.zeros(len(texts), np.uint8), res + res, np.concatenate([decline, decline]))
        done += bits.size
    assert done >= min(N_PATTERNS, 10_000_000) * 0.99
    print(f"\njson_sum: {done} doubles, each as repr and as %.17g")


def _oracle(corpus, handler):
    payloads = [p for p, _ in corpus]
    want = loop.run_task_loop(payloads, [i.to_bytes(4, "little") * 4 for i in range(len(payloads))], handler)
    return payloads, [CODE[w.status] for w in want], [w.result for w in want], [d for _, d in corpus]


@pytest.mark.parametrize("handler", ["json_sum", "identity"])
def test_edge_corpus(queues, handler):
    corpus = sum_edge_payloads() if handler == "json_sum" else value_edge_payloads()
    payloads, st, res, may = _oracle(corpus, handler)
    rec = drain_all(queues[0], payloads, handler)
    declined = check(rec, payloads, st, res, may)
    assert declined >= (sum(may) if handler == "json_sum" else 19)   # the structural limits (and C long) are really declined
    assert_same_records(rec, drain_all(queues[1], payloads, handler), payloads)
    big = [len(p) for p in payloads if len(p) > 48 << 10]
    assert len(big) >= 4 and max(big) >= 512 << 10                     # larger than every stage buffer


def test_llong_min_total(queues):
    p = b'{"args": [{"values": [-9000000000000000000, -220000000000000000, -3372036854775808]}], "kwargs": {}}'
    for q in queues:
        rec = drain_all(q, [p, p.replace(b"-", b"")], "json_sum")
        assert rec.status.tolist() == [0, 4] and rec.result(0) == b"-9223372036854775808"


@pytest.mark.parametrize("handler", ["json_sum", "identity"])
def test_small_ring_partial_drains(handler):
    """Edge payloads inside generated ones, pushed into a 2 MiB ring in small batches and drained a few at a time:
    tiles span pushes, the ring wraps, and identity's deferred value tasks and json_sum's float documents cross both."""
    from beta9_b200 import _lib as L
    from beta9_b200.device_queue import DeviceQueue
    if handler == "json_sum":
        edge, gen = sum_edge_payloads(), synth.json_float_batch(4000, doc_bytes=512, seed=41)
    else:
        edge, gen = value_edge_payloads(), synth.values_batch(8000, seed=42)
    rng = np.random.default_rng(43)
    tasks = [(p, d) for p, d in edge] + [(p, False) for p in gen.tasks()]
    tasks = [tasks[int(i)] for i in rng.permutation(len(tasks))]
    payloads, st, res, may = _oracle(tasks, handler)
    ring_bytes = 2 << 20
    q = DeviceQueue(ring_bytes=ring_bytes, ring_tasks=1 << 12, max_drain_tasks=1 << 12, max_result_bytes=1 << 26)
    try:
        pending = []                                           # task indices, FIFO
        nxt = drains = wraps = 0
        pushed_bytes = 0
        while nxt < len(tasks) or pending:
            if nxt < len(tasks):
                hi, size = nxt, 0
                cap = int(rng.integers(1, 120))
                while hi < len(tasks) and hi - nxt < cap and size + len(payloads[hi]) <= ring_bytes // 2:
                    size += len(payloads[hi])
                    hi += 1
                hi = max(hi, nxt + 1)
                b = synth.from_payloads(payloads[nxt:hi], seed=nxt)
                b.task_ids[:, :4] = np.arange(nxt, hi, dtype=np.uint32).view(np.uint8).reshape(-1, 4)
                try:
                    q.push_batch(b.task_ids, b.payload, b.offsets)
                    pending += range(nxt, hi)
                    pushed_bytes += size
                    nxt = hi
                except L.B9Error as e:
                    assert e.code == L.B9_ENOSPC and pending   # ring full: nothing appended (an empty ring takes any batch)
            take = int(rng.integers(0, 150)) if nxt < len(tasks) else len(pending)
            r = q.drain(handler, max_tasks=take)
            drains += 1
            assert r.n == min(take, len(pending))
            for k in range(r.n):
                i = pending[k]
                assert int(r.task_ids[k, :4].view(np.uint32)[0]) == i
                if int(r.status[k]) == 4 and may[i]:
                    continue
                assert (int(r.status[k]), r.result(k)) == (st[i], res[i]), (payloads[i][:300], int(r.status[k]), r.result(k), res[i])
            pending = pending[r.n:]
        wraps = pushed_bytes // ring_bytes
        assert q.depth() == 0 and q.depth_bytes() == 0
        assert wraps >= 1 and drains >= 50, (wraps, drains)
    finally:
        q.close()
