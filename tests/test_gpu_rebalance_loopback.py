"""b9_rebalance's device half on ONE GPU: W DeviceQueues on device 0 in one worker process, joined by the loopback NCCL
stand-in (tests/loopback_nccl/loopback_nccl.cpp), one thread per rank. Every kernel of the rebalance runs unchanged --
the three byte-prefix scan kernels, rebalance_cut_kernel, both paths of gather_tasks_kernel, ingest_kernel -- as do the
feasibility vote, drop_back / append_segment and the cancelled recount. Only NVLink and NCCL proper stay untested here
(tests/test_gpu_multi.py, two or more GPUs).

References, per case:
* the plan, restated from DESIGN.md section 6 step 3 in integer arithmetic: the pending tasks of all ranks form one
  sequence ordered by (rank, FIFO index); the task whose first byte sits at global position p goes to rank
  min(W - 1, p * W // B). It gives the send matrix -- which must equal b9_rebalance_plan's ranges and the matrix rows
  the ranks all-gathered (read back from the loopback's log) -- and every rank's FIFO afterwards: its kept range, then
  what arrived, source by source in rank order;
* each task's record: oracle.coracle.run_batch for plain SDK payloads, or, for tasks whose carried words matter (flags,
  retries, expiry, TaskMessage / HTTP body / pickle framings), the record an identical twin gets in a queue where it
  never moved."""
import json
import os
import pickle
import signal
import subprocess
import sys

import numpy as np
import pytest

from beta9_b200 import _lib as L
from beta9_b200 import synth
from beta9_b200.device_queue import EXC_BITS, rebalance_plan
from oracle import coracle

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "loopback_nccl", "loopback_nccl.cpp")
WORKER = os.path.join(HERE, "_loopback_rebalance_worker.py")
OP_INIT, OP_ALLGATHER, OP_SEND, OP_RECV = 1, 2, 3, 4
WORKER_TIMEOUT_S = 900
NOW_NS = 1_800_000_000 * 10**9


def build_loopback(out_dir):
    so = os.path.join(str(out_dir), "libloopback_nccl.so")
    r = subprocess.run([os.environ.get("CXX", "g++"), "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, SRC, "-ldl", "-lpthread"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return so


@pytest.fixture(scope="module")
def loopback(tmp_path_factory):
    return build_loopback(tmp_path_factory.mktemp("loopback"))


def run_worker(so, what, tmp_path, env=None):
    """The worker in its own process group, killed with everything it started if it outlives WORKER_TIMEOUT_S."""
    out = os.path.join(str(tmp_path), "out.pkl")
    p = subprocess.Popen([sys.executable, WORKER, so, what, out], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                         env={**os.environ, **(env or {})}, start_new_session=True)
    try:
        log, _ = p.communicate(timeout=WORKER_TIMEOUT_S)
    except subprocess.TimeoutExpired:
        os.killpg(p.pid, signal.SIGKILL)
        log, _ = p.communicate()
        pytest.fail(f"the loopback worker did not finish within {WORKER_TIMEOUT_S} s:\n{log[-4000:]}")
    assert p.returncode == 0, log[-4000:]
    with open(out, "rb") as f:
        return pickle.load(f)


# ---------------------------------------------------------------------------------------------------- the stand-in alone
def test_loopback_alone_against_numpy(loopback, tmp_path):
    got = run_worker(loopback, "selftest", tmp_path, env={"LB_NCCL_TIMEOUT_S": "2"})
    W = 3
    for count in (7, 1000):
        src, res = got[f"allgather_{count}"]
        want = np.concatenate(src)
        for rc, buf in res:
            assert rc == 0 and np.array_equal(buf, want)
    data, res = got["a2a"]
    for r, (rc, rx) in enumerate(res):
        assert rc == 0
        for (s, d, k), v in rx.items():
            assert d == r and np.array_equal(v[:-1], data[(s, d, k)]) and v[-1] == 0     # nothing written past the count
    (rc0, m0), (rc1, m1), (rc2, _) = got["mismatch"]
    assert rc0 != 0 and rc1 != 0 and rc2 == 0
    assert "16 bytes" in m1 and "32 bytes" in m1 and "16 bytes" in m0
    # the log: init, the two AllGathers (the 7-word one with its words), then the Sends / Recvs as posted
    for r, entries in enumerate(got["log"]):
        assert entries[0][:3] == (OP_INIT, -1, W)
        assert entries[1][:3] == (OP_ALLGATHER, -1, 56) and np.array_equal(entries[1][3], got["allgather_7"][0][r])
        assert entries[2][:3] == (OP_ALLGATHER, -1, 1000) and entries[2][3].size == 0
        p2p = [(op, peer, nb) for op, peer, nb, _ in entries[3:3 + 4 * (W - 1)]]
        want_p2p = []
        for d in range(W):
            if d != r:
                for k in range(2):
                    want_p2p += [(OP_SEND, d, len(data[(r, d, k)])), (OP_RECV, d, len(data[(d, r, k)]))]
        assert p2p == want_p2p
    rc, msg = got["unmatched"]
    assert rc != 0 and "no matching Recv" in msg
    rc, msg = got["after_break"]
    assert rc != 0 and "broken" in msg


# ---------------------------------------------------------------------------------------------------- the case model
def plan_dest(lens_per_rank, world):
    """DESIGN.md section 6 step 3, restated: destination rank of every pending task of every rank."""
    total = int(sum(int(l.sum()) for l in lens_per_rank))
    base, out = 0, []
    for l in lens_per_rank:
        pos = base + np.concatenate([[0], np.cumsum(l)[:-1]]).astype(np.int64) if l.size else np.zeros(0, np.int64)
        out.append(np.minimum(world - 1, pos * world // total) if total else np.full(l.size, world - 1, np.int64))
        base += int(l.sum())
    return out


class Case:
    """Steps for the worker and, alongside, what each of them must give."""

    def __init__(self, world, queue=None, queues=None):
        self.W = world
        q = dict(ring_bytes=1 << 20, ring_tasks=1 << 13, max_drain_tasks=1 << 13, max_result_bytes=1 << 22)
        q.update(queue or {})
        self.queue = queues or [dict(q) for _ in range(world)]
        self.batches, self.steps, self.checks = {}, [], []
        self.fifo = [np.zeros(0, np.int64) for _ in range(world)]
        self.ids, self.lens, self.payloads, self.flags, self.exp = [], [], [], [], []
        self.n = 0
        self.expired_at = None

    # -- tasks
    def batch(self, name, b, flags=None, retries=None, ts=None, exp=None):
        n = b.n
        d = {"ids": b.task_ids, "payload": b.payload, "offsets": b.offsets}
        for k, v, dt in (("flags", flags, np.uint8), ("retries", retries, np.uint8), ("ts", ts, np.int64), ("exp", exp, np.int64)):
            if v is not None:
                d[k] = np.asarray(v, dt)
        self.batches[name] = d
        d["base"] = self.n
        self.ids.append(b.task_ids); self.lens.append(np.diff(b.offsets.astype(np.int64))); self.payloads.append(b)
        self.flags.append(np.zeros(n, np.uint8) if flags is None else np.asarray(flags, np.uint8))
        self.exp.append(np.zeros(n, np.int64) if exp is None else np.asarray(exp, np.int64))
        self.n += n
        return name

    def cancel_mask(self):
        """tasks registered so far that carry B9_TF_CANCELLED: pushed so, or expired by an expire step"""
        m = (np.concatenate(self.flags) & L.TF_CANCELLED).astype(bool) if self.flags else np.zeros(0, bool)
        if self.expired_at is not None:
            e = np.concatenate(self.exp)
            m |= (e > 0) & (e <= self.expired_at)
        return m

    def finish_tasks(self):
        self.all_ids = np.concatenate(self.ids) if self.ids else np.zeros((0, 16), np.uint8)
        self.cancelled = self.cancel_mask()

    # -- steps
    def push(self, r, name):
        b = self.batches[name]
        if b["offsets"].shape[0] == 1:
            return
        self.fifo[r] = np.concatenate([self.fifo[r], b["base"] + np.arange(b["offsets"].shape[0] - 1)])
        self.steps.append(("push", r, name))

    def drain(self, tag, handler="identity", max_tasks=None, rank=None):
        ranks = range(self.W) if rank is None else [rank]
        want = []
        for r in ranks:
            k = len(self.fifo[r]) if max_tasks is None else min(max_tasks, len(self.fifo[r]))
            want.append(self.fifo[r][:k][~self.cancel_mask()[self.fifo[r][:k]]])
            self.fifo[r] = self.fifo[r][k:]
        if rank is None:
            self.steps.append(("drain", tag, handler, max_tasks))
        else:
            self.steps.append(("drain_rank", tag, rank, handler, max_tasks))
        self.checks.append(("records", tag, handler, want, rank, "oracle"))

    def peek(self, tag, handler="identity", opts=None, against="oracle"):
        self.steps.append(("peek", tag, handler, opts))
        m = self.cancel_mask()
        self.checks.append(("records", tag, handler, [f[~m[f]] for f in self.fifo], None, against))

    def rebalance(self, tag, refused=False):
        W = self.W
        all_lens = np.concatenate(self.lens) if self.lens else np.zeros(0, np.int64)
        lens = [all_lens[f] for f in self.fifo]
        m = self.cancel_mask()
        cancelled = [int(m[f].sum()) for f in self.fifo]
        dest = plan_dest(lens, W)
        M = np.zeros((W, W, 2), np.int64)
        for s in range(W):
            for d in range(W):
                m = dest[s] == d
                M[s, d] = (int(m.sum()), int(lens[s][m].sum()))
        before = [f.copy() for f in self.fifo]
        if not refused:
            self.fifo = [np.concatenate([before[d][dest[d] == d]] + [before[s][dest[s] == d] for s in range(W) if s != d]) for d in range(W)]
        self.steps.append(("rebalance", tag))
        self.checks.append(("rebalance", tag, before, lens, cancelled, M, refused))

    def expire(self, tag, now_ns):
        was = self.cancel_mask()
        self.expired_at = now_ns
        newly = self.cancel_mask() & ~was
        want = [int(newly[f].sum()) for f in self.fifo]
        self.steps.append(("expire", tag, now_ns))
        self.checks.append(("equal", tag, want))


def oracle_table(case, handler):
    """status, has, result offsets and bytes of every task of the case under coracle."""
    b = synth.concat(case.payloads) if len(case.payloads) > 1 else case.payloads[0]
    o = coracle.run_batch(b.task_ids, b.payload, b.offsets, handler)
    return o.status, o.has, o.offsets.astype(np.int64), o.payload


def twin_table(case, twin):
    """the same, from the PEEK records of a twin queue (tasks it did not give a record to: status 255)"""
    status = np.full(case.n, 255, np.uint8)
    has = np.zeros(case.n, np.uint8)
    lens = np.zeros(case.n, np.int64)
    key = {case.all_ids[i].tobytes(): i for i in range(case.n)}
    idx = np.array([key[twin["ids"][j].tobytes()] for j in range(len(twin["status"]))], np.int64)
    status[idx] = twin["status"]; has[idx] = twin["has"]; lens[idx] = twin["lens"]
    off = np.zeros(case.n + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    blob = np.zeros(int(off[-1]), np.uint8)
    src = np.concatenate([[0], np.cumsum(twin["lens"].astype(np.int64))])
    for j, i in enumerate(idx):
        blob[off[i]:off[i + 1]] = twin["payload"][src[j]:src[j + 1]]
    return status, has, off, blob


def gather(blob, off, idx):
    """bytes of records idx, back to back"""
    ln = off[idx + 1] - off[idx]
    if not ln.size or not ln.sum():
        return np.zeros(0, np.uint8)
    ends = np.cumsum(ln)
    rec = np.repeat(np.arange(idx.size), ln)
    pos = off[idx][rec] + (np.arange(int(ends[-1])) - (ends - ln)[rec])
    return blob[pos]


def check_records(case, got, handler, want_fifo, table):
    status, has, off, blob = table
    live = want_fifo
    assert got["ids"].shape[0] == live.size, (got["ids"].shape[0], live.size)
    assert np.array_equal(got["ids"], case.all_ids[live]), "records out of the expected FIFO order"
    assert status[live].max(initial=0) != 255, "a task the twin did not answer"
    bad = np.nonzero((got["status"] != status[live]) | (got["has"] != has[live]))[0]
    assert bad.size == 0, f"{bad.size} records differ, first at FIFO position {bad[:1]}: status {got['status'][bad[:3]]} against {status[live][bad[:3]]}"
    want_bytes = gather(blob, off, live[has[live] != 0])
    got_bytes = gather(got["payload"], np.concatenate([[0], np.cumsum(got["lens"].astype(np.int64))]), np.nonzero(got["has"])[0])
    assert np.array_equal(got_bytes, want_bytes), "result bytes differ"


def run_case(case, loopback, tmp_path):
    case.finish_tasks()
    cp = os.path.join(str(tmp_path), "case.pkl")
    with open(cp, "wb") as f:
        pickle.dump({"world": case.W, "queue": case.queue, "batches": {k: {kk: vv for kk, vv in v.items() if kk != "base"} for k, v in case.batches.items()},
                     "steps": case.steps}, f)
    out = run_worker(loopback, cp, tmp_path)
    tables = {}
    for chk in case.checks:
        kind, tag = chk[0], chk[1]
        if kind == "equal":
            assert out[tag] == chk[2], (tag, out[tag], chk[2])
        elif kind == "records":
            _, _, handler, want, rank, against = chk
            if against == "oracle":
                if handler not in tables:
                    tables[handler] = oracle_table(case, handler)
                table = tables[handler]
            else:
                twin_tag, k = against
                table = twin_table(case, out[twin_tag]["drains"][k])
            if rank is not None:
                check_records(case, out[tag], handler, want[0], table)
            else:
                for r in range(case.W):
                    check_records(case, out[tag][r], handler, want[r], table)
                ids = np.concatenate([out[tag][r]["ids"] for r in range(case.W)])      # every task exactly once over the ranks
                assert len({bytes(x) for x in ids}) == ids.shape[0] == sum(len(w) for w in want)
        elif kind == "rebalance":
            check_rebalance(case, out[tag], *chk[2:])
    return out


def check_matrix_rows(got, M):
    """each rank's row of the send matrix, as the ranks all-gathered it (the loopback's log), against M [W, W, 2]"""
    for r, g in enumerate(got):
        ag = [e for e in g["log"] if e[0] == OP_ALLGATHER]
        assert len(ag) == 3, [e[:3] for e in g["log"]]
        assert np.array_equal(ag[1][3].astype(np.int64), M[r].reshape(-1)), (r, ag[1][3], M[r].reshape(-1))


def check_rebalance(case, got, before, lens, cancelled, M, refused):
    W = case.W
    dest = plan_dest(lens, W)
    counts = np.array([len(f) for f in before], np.uint64)
    nbytes = np.array([int(l.sum()) for l in lens], np.uint64)
    for r in range(W):
        g = got[r]
        if refused:
            assert g["rc"] == L.B9_ENOSPC, (r, g["rc"], g["info"])
            assert (g["depth"], g["depth_bytes"]) == (int(counts[r]), int(nbytes[r]))
            assert not [e for e in g["log"] if e[0] in (OP_SEND, OP_RECV)], "a refused exchange moved data"
            continue
        assert g["rc"] == 0, (r, g["info"])
    if refused:
        return
    check_matrix_rows(got, M)
    for r in range(W):
        g = got[r]
        # the library's own plan over the same prefix gives the same ranges as the restated one
        prefix = np.concatenate([[0], np.cumsum(lens[r])]).astype(np.uint64)
        lo, hi = rebalance_plan(W, r, counts, nbytes, prefix)
        for d in range(W):
            idx = np.nonzero(dest[r] == d)[0]
            if idx.size:
                assert (int(lo[d]), int(hi[d])) == (int(idx[0]), int(idx[-1]) + 1), (r, d)
            else:
                assert int(lo[d]) == int(hi[d]), (r, d)
        sent = M[r, :, :].sum(axis=0) - M[r, r]
        recv = M[:, r, :].sum(axis=0) - M[r, r]
        after = M[:, r, :].sum(axis=0)
        assert tuple(int(x) for x in g["info"]) == (int(counts[r]), int(nbytes[r]), int(sent[0]), int(sent[1]), int(recv[0]), int(recv[1]),
                                                    int(after[0]), int(after[1])), (r, g["info"])
        assert (g["depth"], g["depth_bytes"]) == (int(after[0]), int(after[1]))
        # the loopback's log: (count, bytes, cancelled, 0), then this rank's matrix row, then the vote; the payload sends
        ag = [e for e in g["log"] if e[0] == OP_ALLGATHER]
        assert len(ag) == 3, [e[:3] for e in g["log"]]
        assert [int(x) for x in ag[0][3]] == [int(counts[r]), int(nbytes[r]), cancelled[r], 0]
        assert [int(x) for x in ag[2][3]] == [1]
        for d in range(W):
            if d == r:
                continue
            sends = [e[2] for e in g["log"] if e[0] == OP_SEND and e[1] == d]
            recvs = [e[2] for e in g["log"] if e[0] == OP_RECV and e[1] == d]
            assert len(sends) == (0 if not M[r, d, 0] else 1 if not M[r, d, 1] else 2)
            assert len(recvs) == (0 if not M[d, r, 0] else 1 if not M[d, r, 1] else 2)
            if M[r, d, 1]:
                assert sends[1] == M[r, d, 1]
            if M[d, r, 1]:
                assert recvs[1] == M[d, r, 1]


# ---------------------------------------------------------------------------------------------------- task builders
_seed = [1000]


def plain(n, chars=None, lengths=None):
    """n identity tasks with one string argument; ids unique over the whole module"""
    _seed[0] += 1
    if n == 0:
        return synth.Batch(np.zeros((0, 16), np.uint8), np.zeros(0, np.uint8), np.zeros(1, np.uint64))
    if chars is not None:
        b = synth.strings_batch(n, chars, adversarial_frac=0.0, seed=_seed[0])
    else:
        if lengths is None:
            lengths = np.random.default_rng(_seed[0]).integers(1, 400, n)
        b = synth.crc_batch(n, seed=_seed[0], lengths=np.full(n, lengths) if np.isscalar(lengths) else lengths)
    b.task_ids = synth.task_ids(n, seed=_seed[0])
    return b


def sound_ring(case, tag):
    """after the exchange: a popping drain of everything, a new push on every rank, a drain -- all as the oracle says"""
    case.drain(f"{tag}_all")
    for r in range(case.W):
        case.push(r, case.batch(f"{tag}_again{r}", plain(37 + 5 * r, lengths=30)))
    case.drain(f"{tag}_again")


def skewed(W, heavy, light, one_push=True):
    c = Case(W)
    for r in range(W):
        n = heavy if r == 0 else light
        if one_push or n < 8:
            c.push(r, c.batch(f"r{r}", plain(n)))
        else:
            b = plain(n)
            k = max(1, n // 7)
            for i, lo in enumerate(range(0, n, k)):
                c.push(r, c.batch(f"r{r}_{i}", b.slice(lo, min(n, lo + k))))
    return c


def case_skew(W):
    c = skewed(W, 2400, 150)
    c.rebalance("reb")
    c.peek("peek")
    sound_ring(c, "s")
    return c


def case_rank0_only():
    c = skewed(3, 3000, 0)                     # every cut inside rank 0's one segment: a partial drop_back
    c.rebalance("reb")
    c.peek("peek")
    sound_ring(c, "s")
    return c


def case_last_empty():
    c = Case(4)
    for r in range(3):
        c.push(r, c.batch(f"r{r}", plain(500 + 300 * r)))
    c.rebalance("reb")
    c.peek("peek")
    sound_ring(c, "s")
    return c


def case_max_world():
    W = 16
    c = Case(W, queue=dict(ring_bytes=1 << 19, ring_tasks=1 << 12, max_drain_tasks=1 << 12, max_result_bytes=1 << 21))
    rng = np.random.default_rng(16)
    for r in range(W):
        n = 1500 if r == 0 else int(rng.integers(0, 120)) * (r % 5 != 3)
        c.push(r, c.batch(f"r{r}", plain(n)))
    c.rebalance("reb")
    c.peek("peek")
    sound_ring(c, "s")
    return c


def case_all_empty():
    c = Case(3)
    c.rebalance("reb")
    c.peek("peek")
    sound_ring(c, "s")
    return c


def case_balanced():
    c = Case(4)
    for r in range(4):
        c.push(r, c.batch(f"r{r}", plain(300, chars=40)))     # equal counts of equal lengths: every task already where it belongs
    c.rebalance("reb")
    c.peek("peek")
    return c


def case_big_task():
    c = Case(2)
    c.push(0, c.batch("small0", plain(20, lengths=100)))
    c.push(0, c.batch("big", plain(1, lengths=30000)))       # more than B / W on its own
    c.push(0, c.batch("small1", plain(20, lengths=100)))
    c.push(1, c.batch("r1", plain(5, lengths=50)))
    c.rebalance("reb")
    c.peek("peek")
    sound_ring(c, "s")
    return c


def case_scan_blocks(counts):
    c = Case(len(counts), queue=dict(ring_bytes=1 << 21))
    for r, n in enumerate(counts):
        c.push(r, c.batch(f"r{r}", plain(n, lengths=np.random.default_rng(n).integers(1, 60, max(n, 1))[:n])))
    c.rebalance("reb")
    c.peek("peek")
    sound_ring(c, "s")
    return c


def case_million():
    n = 1024 * 1024 + 4099                    # 1029 scan blocks: scan_of_sums_kernel walks 2 block sums per thread
    q = dict(ring_bytes=1 << 26, ring_tasks=1 << 21, max_drain_tasks=1 << 21, max_result_bytes=1 << 27)
    c = Case(2, queue=q)
    c.push(0, c.batch("big", plain(n, lengths=np.random.default_rng(3).integers(1, 12, n))))
    c.push(1, c.batch("r1", plain(1000, lengths=8)))
    c.rebalance("reb")
    c.peek("peek")
    return c


def case_wrap_slots():
    c = Case(2, queue=dict(ring_tasks=1024, max_drain_tasks=1024))
    c.push(0, c.batch("first", plain(1000, lengths=20)))
    c.drain("first_out", rank=0)
    c.push(0, c.batch("wrapped", plain(900, lengths=20)))      # slots 1000 .. 1899: past slot_mask and round
    c.push(1, c.batch("r1", plain(40, lengths=20)))
    c.rebalance("reb")
    c.peek("peek")
    sound_ring(c, "s")
    return c


def case_wrap_bytes():
    """rank 0's FIFO = segment B (end of the byte ring) then C (placed back at 0) then many small pushes: ranges that
    leave span segments and the wrap, so they go through the staged, warp-per-task gather"""
    c = Case(3, queues=[dict(ring_bytes=1 << 16, ring_tasks=1 << 12, max_drain_tasks=1 << 12, max_result_bytes=1 << 22)] +
             [dict(ring_bytes=1 << 20, ring_tasks=1 << 12, max_drain_tasks=1 << 12, max_result_bytes=1 << 22) for _ in range(2)])
    c.push(0, c.batch("A", plain(200, lengths=100)))          # ~24 KiB
    c.push(0, c.batch("B", plain(200, lengths=100)))
    c.drain("A_out", max_tasks=200, rank=0)
    c.push(0, c.batch("C", plain(120, lengths=100)))          # does not fit after B: placed at 0
    for i in range(6):
        c.push(0, c.batch(f"D{i}", plain(3, lengths=60)))
    c.push(1, c.batch("r1", plain(10, lengths=90)))
    c.rebalance("reb")
    c.peek("peek")
    sound_ring(c, "s")
    return c


def case_many_pushes():
    c = skewed(3, 2100, 90, one_push=False)
    c.rebalance("reb")
    c.peek("peek")
    sound_ring(c, "s")
    return c


def case_twice():
    c = skewed(3, 1800, 100)
    c.rebalance("reb1")
    c.drain("half", max_tasks=300)
    c.push(2, c.batch("more", plain(900)))
    c.rebalance("reb2")
    c.rebalance("reb3")                       # already balanced: nothing moves
    c.peek("peek")
    sound_ring(c, "s")
    return c


def case_enospc():
    c = Case(3, queues=[dict(ring_bytes=1 << 20, ring_tasks=1 << 13, max_drain_tasks=1 << 13, max_result_bytes=1 << 22) for _ in range(2)] +
             [dict(ring_bytes=1 << 12, ring_tasks=1 << 13, max_drain_tasks=1 << 13, max_result_bytes=1 << 22)])
    c.push(0, c.batch("r0", plain(2000, lengths=40)))
    c.push(2, c.batch("r2", plain(3, lengths=40)))
    c.peek("before")
    c.rebalance("reb", refused=True)
    c.peek("after")
    sound_ring(c, "s")
    return c


def case_peek_waiting():
    c = skewed(2, 1200, 50)
    c.steps.append(("peek_launch", "identity"))
    c.rebalance("reb")
    c.steps.append(("fetch", "fetch_after"))
    c.checks.append(("equal", "fetch_after", [L.B9_EINVAL, L.B9_EINVAL]))
    c.peek("peek")
    sound_ring(c, "s")
    return c


def case_carried_words():
    """Tasks whose carried words change their record: retries under a policy, expiry, cancelled slots, TaskMessage /
    HTTP body / pickle framings. Each is compared with its twin in a queue where it never moved."""
    import uuid

    from oracle.pyoracle import loop
    from oracle.pyoracle.loop import sdk_put_payload
    from tests import pickle_corpus
    W = 3
    c = Case(W)
    payloads, flags, retries, ts, exp = [], [], [], [], []
    rng = np.random.default_rng(77)

    def add(p, f=0, rt=0):
        payloads.append(p); flags.append(f); retries.append(rt)
        k = len(ts)
        ts.append(1_700_000_000 + k)
        exp.append([0, NOW_NS - 1000 - k, NOW_NS + 10**12 + k][int(rng.integers(0, 3))])
    for k in range(60):
        add(sdk_put_payload(f"v{k}"))
        add(sdk_put_payload(), 0, k % 4)                                   # TypeError: RETRY below 2 retries, RETRY_LIMIT from 2
        add(json.dumps({"args": [f"h{k}"]}).encode(), L.TF_HTTP_BODY)
        add(sdk_put_payload(f"c{k}"), L.TF_CANCELLED)
    blobs = pickle_corpus.sdk_blobs(20)[:60]
    for b in blobs:
        add(b, L.TF_PICKLE)
    n_plain = len(payloads)
    msg_ids = [uuid.UUID(int=(0xB9 << 100) | k).bytes for k in range(40)]
    wires = loop.run_task_loop([sdk_put_payload(f"m{k}") for k in range(40)], msg_ids, "identity", keep_wire=True)
    for w in wires:
        add(w.wire, L.TF_TASK_MSG)
    order = rng.permutation(len(payloads))
    ids = synth.task_ids(len(payloads), seed=4242)
    for j in range(40):
        ids[n_plain + j] = np.frombuffer(msg_ids[j], np.uint8)
    b = synth.from_payloads([payloads[i] for i in order])
    b.task_ids = ids[order]
    sel = lambda a: np.asarray(a)[order]                                    # noqa: E731
    f, rt, t, e = sel(flags), sel(retries), sel(ts), sel(exp)
    n = b.n
    c.push(0, c.batch("heavy", b.slice(0, n - 40), flags=f[:n - 40], retries=rt[:n - 40], ts=t[:n - 40], exp=e[:n - 40]))
    c.push(1, c.batch("light", b.slice(n - 40, n), flags=f[n - 40:], retries=rt[n - 40:], ts=t[n - 40:], exp=e[n - 40:]))
    mask = EXC_BITS[TypeError]
    c.steps.append(("policy", mask, 2))
    c.rebalance("reb")
    c.expire("expired", NOW_NS)
    drains = [("identity", None), ("identity", {"full_pickle": True}), ("identity", {"endpoint": True}), ("crc32", None)]
    c.steps.append(("twin", "twin", ["heavy", "light"], (mask, 2), NOW_NS, drains))
    c.checks.append(("twin_expired", "twin"))
    for k, (h, opts) in enumerate(drains):
        c.peek(f"peek{k}", h, opts, against=("twin", k))
    return c


CASES = {
    "skew_w2": lambda: case_skew(2),
    "skew_w3": lambda: case_skew(3),
    "skew_w4": lambda: case_skew(4),
    "rank0_only_w3": case_rank0_only,
    "last_empty_w4": case_last_empty,
    "max_world_w16": case_max_world,
    "all_empty_w3": case_all_empty,
    "balanced_w4": case_balanced,
    "big_task_w2": case_big_task,
    "scan_blocks_w4": lambda: case_scan_blocks([1023, 1024, 1025, 4097]),
    "scan_blocks_w3": lambda: case_scan_blocks([1, 4097, 0]),
    "million_w2": case_million,
    "wrap_slots_w2": case_wrap_slots,
    "wrap_bytes_w3": case_wrap_bytes,
    "many_pushes_w3": case_many_pushes,
    "twice_w3": case_twice,
    "enospc_w3": case_enospc,
    "peek_waiting_w2": case_peek_waiting,
    "carried_words_w3": case_carried_words,
}


@pytest.mark.parametrize("name", list(CASES))
def test_rebalance_loopback(name, loopback, tmp_path):
    case = CASES[name]()
    out = run_case(case, loopback, tmp_path)
    for chk in case.checks:
        if chk[0] == "twin_expired":
            assert out[chk[1]]["expired"] == sum(out["expired"])
    if name == "balanced_w4":
        for g in out["reb"]:
            assert not [e for e in g["log"] if e[0] in (OP_SEND, OP_RECV)]


def test_matrix_check_fails_on_a_prefix_one_task_off(loopback, tmp_path):
    """The matrix check is not vacuous: the rows the ranks all-gathered match the matrix of the true prefixes, and
    fail against the matrix of rank 0's prefix with its first task left out."""
    case = skewed(2, 600, 40)
    case.rebalance("reb")
    out = run_case(case, loopback, tmp_path)
    _, _, before, lens, _, M, _ = case.checks[-1]
    check_matrix_rows(out["reb"], M)
    off = [lens[0][1:], lens[1]]
    dest = plan_dest(off, 2)
    M_off = np.zeros((2, 2, 2), np.int64)
    for s in range(2):
        for d in range(2):
            m = dest[s] == d
            M_off[s, d] = (int(m.sum()), int(off[s][m].sum()))
    assert not np.array_equal(M_off, M)
    with pytest.raises(AssertionError):
        check_matrix_rows(out["reb"], M_off)
