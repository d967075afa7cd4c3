"""GPU: every way drain3_kernel reads a task's bytes, for every handler, against plain references.

tests/stage_corpus.py builds the corpora and restates how the kernel stages a warp-tile (its module docstring lists
the four ways); tests/test_stage_corpus_on_host.py checks their expectations against the oracle on the CPU.
- lane-boundary strings (identity, crc32): escapes, surrogate pairs and raw UTF-8 at every offset around the starts
  of lane chunks 1, 15 and 31, for chunk sizes of 1 to 40 000 bytes; the large ones are read from the ring (way 3);
- mixed windows (every handler): small tasks with runs of medium ones and a few of 2 KiB to 1 MiB (ways 1, 2, 3);
- tiles of exactly the stage buffer's size and 16 bytes either side, contiguous and scattered (ways 1, 2, 4);
- pushes and partial drains on a 1 MiB ring, where tiles span pushes and the ring's wrap (way 4 staged and refused);
- crc32 bodies of up to 48 MB whose lanes' zero-shifts set every bit 0..25.
Each runs on a queue with the window's own stage buffer and on one with a 1 KiB buffer (B9_STAGE_BYTES=1024), and
each also with a few cancelled slots, where the record index comes from the count pre-pass (tile_count_kernel).
Records must equal the reference, or the oracle where there is none (lone surrogates, invalid UTF-8). None of these
tasks may be declined (B9_ST_UNSUPPORTED): include/b9gpu.h declines only number literals, nesting and member counts."""
import os

import numpy as np
import pytest

from beta9_b200 import synth
from oracle import coracle
from tests import stage_corpus as sc

pytestmark = pytest.mark.gpu
CANCEL_EVERY = 53                                    # count mode: slots i % 53 == 7 are pushed cancelled
MAX_PUSH_BYTES = 96 << 20


def _queue(stage: int = 0, **kw):
    from beta9_b200.device_queue import DeviceQueue
    old = os.environ.get("B9_STAGE_BYTES")
    if stage:
        os.environ["B9_STAGE_BYTES"] = str(stage)
    try:
        return DeviceQueue(**kw)
    finally:
        if old is None:
            os.environ.pop("B9_STAGE_BYTES", None)
        else:
            os.environ["B9_STAGE_BYTES"] = old


@pytest.fixture(scope="module")
def queues():
    """The window's own stage buffer, and a 1 KiB one; tasks of up to 4 MiB (the mixed windows hold 1 MiB tasks)."""
    kw = dict(ring_bytes=256 << 20, ring_tasks=1 << 16, max_drain_tasks=1 << 16, max_result_bytes=256 << 20, max_task_bytes=4 << 20)
    qs = {0: _queue(**kw), 1024: _queue(1024, **kw)}
    yield qs
    for q in qs.values():
        q.close()


@pytest.fixture(scope="module")
def big_queue():
    """Room for the largest crc32 body (48 MB)."""
    q = _queue(ring_bytes=128 << 20, ring_tasks=1 << 10, max_drain_tasks=1 << 10, max_result_bytes=1 << 20, max_task_bytes=64 << 20)
    yield q
    q.close()


def cancel_mask(n: int, count_mode: bool) -> np.ndarray:
    m = np.zeros(n, bool)
    if count_mode:
        m[7::CANCEL_EVERY] = True
        m[n - 1] = n > 1                              # a cancelled slot in the last tile too
    return m


def run(q, c: sc.Corpus, cancelled: np.ndarray, window: int = 4000):
    """Push the corpus into an empty queue and drain it, `window` tasks (and at most MAX_PUSH_BYTES) at a time.
    Returns the records of the tasks that were not cancelled, in task order."""
    out = []
    lo = 0
    while lo < c.n:
        hi, size = lo, 0
        while hi < c.n and hi - lo < window and (hi == lo or size + len(c.payloads[hi]) <= MAX_PUSH_BYTES):
            size += len(c.payloads[hi])
            hi += 1
        b = synth.from_payloads(c.payloads[lo:hi], seed=lo)
        assert q.depth() == 0
        q.push_batch(b.task_ids, b.payload, b.offsets, flags=cancelled[lo:hi].astype(np.uint8))
        r = q.drain(c.handler, max_tasks=b.n)
        keep = np.flatnonzero(~cancelled[lo:hi])
        assert r.n_popped == b.n and r.n == keep.size and q.depth() == 0
        assert np.array_equal(r.task_ids, b.task_ids[keep])
        out += [(int(r.status[i]), r.result(i)) for i in range(r.n)]
        lo = hi
    return out


def expected(c: sc.Corpus):
    """The reference's record, or the oracle's (run with every CPU thread) where the corpus has none."""
    want = list(c.want)
    todo = [i for i, w in enumerate(want) if w is None]
    if todo:
        b = synth.from_payloads([c.payloads[i] for i in todo], seed=3)
        o = coracle.run_batch(b.task_ids, b.payload, b.offsets, c.handler, nthreads=os.cpu_count() or 1)
        for k, i in enumerate(todo):
            want[i] = (int(o.status[k]), o.result(k))
    return want


def check(q, c: sc.Corpus, want, count_mode: bool, window: int = 4000):
    cancelled = cancel_mask(c.n, count_mode)
    got = run(q, c, cancelled, window)
    keep = np.flatnonzero(~cancelled).tolist()
    declined = [i for i, g in zip(keep, got) if g[0] == 4]
    assert not declined, ("declined", len(declined), c.payloads[declined[0]][:300])
    bad = [i for i, g in zip(keep, got) if g != want[i]]
    if bad:
        i = bad[0]
        g = got[keep.index(i)]
        raise AssertionError((len(bad), len(c.payloads[i]), c.payloads[i][:300], g[0], (g[1] or b"")[:300], want[i][0], (want[i][1] or b"")[:300]))


@pytest.fixture(scope="module")
def lane_corpora():
    out = {}
    for h in ("identity", "crc32"):
        c = sc.lane_boundary_strings(h)
        out[h] = (c, expected(c))
    return out


@pytest.mark.parametrize("count_mode", [False, True], ids=["plain", "count"])
@pytest.mark.parametrize("stage", [0, 1024], ids=["stage_window", "stage_1k"])
@pytest.mark.parametrize("handler", ["identity", "crc32"])
def test_lane_boundary_strings(queues, lane_corpora, handler, stage, count_mode):
    c, want = lane_corpora[handler]
    check(queues[stage], c, want, count_mode)


@pytest.mark.parametrize("count_mode", [False, True], ids=["plain", "count"])
@pytest.mark.parametrize("stage", [0, 1024], ids=["stage_window", "stage_1k"])
@pytest.mark.parametrize("handler", ["identity", "crc32", "vadd_f32", "json_sum"])
def test_mixed_windows(queues, handler, stage, count_mode):
    c = sc.mixed_windows(handler, seed=int(count_mode))
    check(queues[stage], c, expected(c), count_mode)


@pytest.mark.parametrize("count_mode", [False, True], ids=["plain", "count"])
@pytest.mark.parametrize("stage", [0, 1024], ids=["stage_window", "stage_1k"])
@pytest.mark.parametrize("handler", ["identity", "crc32", "vadd_f32", "json_sum"])
def test_exact_fit_tiles(queues, handler, stage, count_mode):
    q = queues[stage]
    for w in sc.exact_fit_tiles(handler):
        c = w.corpus
        cancelled = cancel_mask(c.n, count_mode)
        lo = 0
        for n in w.pushes:                            # the second push of a scattered window starts at the next 256 bytes
            b = synth.from_payloads(c.payloads[lo:lo + n], seed=lo)
            q.push_batch(b.task_ids, b.payload, b.offsets, flags=cancelled[lo:lo + n].astype(np.uint8))
            lo += n
        r = q.drain(handler, max_tasks=c.n)
        keep = np.flatnonzero(~cancelled).tolist()
        assert r.n_popped == c.n and r.n == len(keep) and q.depth() == 0
        assert [(int(r.status[k]), r.result(k)) for k in range(r.n)] == [c.want[i] for i in keep], (w.target, w.scattered)


@pytest.mark.parametrize("count_mode", [False, True], ids=["plain", "count"])
@pytest.mark.parametrize("stage", [0, 1024], ids=["stage_window", "stage_1k"])
@pytest.mark.parametrize("handler", ["crc32", "vadd_f32", "json_sum"])
def test_ring_wrap(handler, stage, count_mode):
    """Pushes of 1..119 tasks (never a multiple of the tile size) and drains of 0..59 on a 1 MiB ring. RingModel
    (ring_place.h's rule) predicts where every push lands; a push the model refuses must be refused by the queue and the
    other way round. From those offsets: tiles that span pushes are read as scattered tiles, some of them across the
    ring's wrap, and with the 1 KiB buffer some scattered tiles are refused and read from the ring."""
    from beta9_b200 import _lib as L
    src = sc.mixed_windows(handler, seed=10 + int(count_mode), n_small=20000)
    src.extend(sc.mixed_windows(handler, seed=30 + int(count_mode), n_small=20000))     # about four passes over the ring
    tasks = [i for i, p in enumerate(src.payloads) if len(p) <= 160 << 10]
    payloads = [src.payloads[i] for i in tasks]
    want = [src.want[i] for i in tasks]
    cancelled = cancel_mask(len(payloads), count_mode)
    ring = 1 << 20
    q = _queue(stage, ring_bytes=ring, ring_tasks=1 << 16, max_drain_tasks=1 << 13, max_result_bytes=1 << 26, max_task_bytes=1 << 20)
    model = sc.RingModel(ring)
    rng = np.random.default_rng(20 + stage + int(count_mode))
    T = sc.T_OF[handler]
    paths = {"1": 0, "2": 0, "3": 0, "4": 0, "4r": 0, "fit": 0}
    wrap_tiles = drains = refused = 0
    pending = []
    nxt = 0
    try:
        while nxt < len(payloads) or pending:
            if nxt < len(payloads):
                k = int(rng.integers(1, 120))
                k += k % T == 0
                hi = min(len(payloads), nxt + k)
                lens = [len(p) for p in payloads[nxt:hi]]
                start = model.push(lens)
                b = synth.from_payloads(payloads[nxt:hi], seed=nxt)
                b.task_ids[:, :4] = np.arange(nxt, hi, dtype=np.uint32).view(np.uint8).reshape(-1, 4)
                try:
                    q.push_batch(b.task_ids, b.payload, b.offsets, flags=cancelled[nxt:hi].astype(np.uint8))
                    assert start is not None, "the queue took a push that ring_place.h refuses"
                    pending += range(nxt, hi)
                    nxt = hi
                except L.B9Error as e:
                    assert e.code == L.B9_ENOSPC and start is None, (e.code, start)
                    refused += 1
            take = min(int(rng.integers(0, 60)) if nxt < len(payloads) else 150, len(pending))
            if take:
                offs, lens, max_len = model.window(take)
                tt = sc.tile_tasks(handler, take)
                cap = sc.stage_cap(handler, take, sum(lens), max_len, stage)
                for key, v in sc.read_paths(offs, lens, tt, cap).items():
                    paths[key] += v
                wrap_tiles += sum(any(offs[j] < offs[j - 1] for j in range(t0 + 1, min(take, t0 + tt))) for t0 in range(0, take, tt))
            r = q.drain(handler, max_tasks=take)
            drains += 1
            got = [i for i in pending[:take] if not cancelled[i]]
            assert r.n_popped == take and r.n == len(got)
            for k, i in enumerate(got):
                assert int(r.task_ids[k, :4].view(np.uint32)[0]) == i
                assert (int(r.status[k]), r.result(k)) == want[i], (len(payloads[i]), payloads[i][:200], int(r.status[k]), r.result(k), want[i])
            model.pop(take)
            pending = pending[take:]
        assert q.depth() == 0 and model.depth() == 0
    finally:
        q.close()
    assert refused > 0 and wrap_tiles > 0 and paths["4"] > 0, (refused, wrap_tiles, paths)
    assert paths["4r"] > 0 or not stage, paths
    print(f"\n{handler} stage={stage or 'window'}: {drains} drains, {refused} pushes refused, {wrap_tiles} tiles across the wrap, {paths}")


@pytest.mark.parametrize("count_mode", [False, True], ids=["plain", "count"])
def test_crc_shift_levels(big_queue, count_mode):
    c = sc.crc_shift_levels()
    if count_mode:                                    # small cancelled tasks between the bodies
        d = sc.Corpus("crc32")
        for p, w in zip(c.payloads, c.want):
            d.add(sc.framed(b"x"), sc.ref_crc32("x"))
            d.add(p, w)
        c = d
    cancelled = np.zeros(c.n, bool)
    if count_mode:
        cancelled[0::2] = True
    got = run(big_queue, c, cancelled, window=c.n)
    keep = np.flatnonzero(~cancelled).tolist()
    for i, g in zip(keep, got):
        assert g == c.want[i], (len(c.payloads[i]), g, c.want[i])
