"""The expectations of tests/test_gpu_stage_paths.py, checked on the CPU before they are used on the GPU.

For every task of every builder of tests/stage_corpus.py, the independent reference (json / zlib / numpy / sum) must
equal the oracle: the C task loop (coracle) for every task, and the Python task loop (pyoracle) for every task of up to
64 KiB (above that its per-character Go decoder takes seconds per task; test_oracle_c_vs_py.py pins the two oracles
against each other). Tasks without a reference (lone surrogates, invalid UTF-8) must get the same record from both
oracles. The builders' coverage assertions run here too, and the restatements of the kernel's staging choices and of
the ring's placement rule are checked: the former on the corpora (which ways they reach), the latter against
ring_place.h compiled for the host."""
import os

import numpy as np
import pytest

from beta9_b200 import synth
from oracle import coracle
from oracle.pyoracle import loop
from tests import stage_corpus as sc
from tests.test_ring_place import POP, PUSH, script  # noqa: F401  (the ring_place.h host build, as a fixture)

CODE = {"COMPLETE": 0, "ERROR": 1, "RETRY": 2, "REJECTED": 3}
PY_MAX = 64 << 10


def check_against_oracles(c: sc.Corpus) -> int:
    b = synth.from_payloads(c.payloads, seed=5)
    o = coracle.run_batch(b.task_ids, b.payload, b.offsets, c.handler, nthreads=os.cpu_count() or 1)
    got = [(int(o.status[i]), o.result(i)) for i in range(c.n)]
    for i, w in enumerate(c.want):
        if w is not None:
            assert got[i] == w, (c.payloads[i][:200], got[i], w)
    small = [i for i, p in enumerate(c.payloads) if len(p) <= PY_MAX]
    py = loop.run_task_loop([c.payloads[i] for i in small], [b.task_ids[i].tobytes() for i in small], c.handler)
    for i, r in zip(small, py):
        assert (CODE[r.status], r.result) == got[i], (c.payloads[i][:200], r.status, r.result, got[i])
    return len(small)


def test_lane_coverage_and_shift_bits():
    cov = sc.lane_coverage_expected()
    for S in sc.LANE_S:                                             # every unit at some offset of every lane start
        assert {(name, k) for s, name, k, d in cov if s == S} == {(name, k) for name in sc.UNITS for k in sc.LANE_KS
                                                                    if k * S - 6 + len(sc.UNITS[name]) <= 32 * S}
    bits = 0
    for n in sc.SHIFT_N:
        for sh in sc.lane_shifts(n):
            bits |= sh
    assert all(bits >> k & 1 for k in range(sc.SHIFT_BITS))
    assert sc.lane_shifts(32 * 1000)[0] == 31 * 1000 and sc.lane_shifts(10) == [9, 8, 7, 6, 5, 4, 3, 2, 1] + [0] * 23


@pytest.mark.parametrize("handler", ["identity", "crc32"])
def test_lane_boundary_strings(handler):
    c = sc.lane_boundary_strings(handler)
    n_py = check_against_oracles(c)
    assert n_py >= c.n - 200
    assert sum(w is None for w in c.want) >= 5 * len(sc.LANE_S) * 13        # the Go-only units really are oracle-only
    assert max(len(p) for p in c.payloads) > 48 << 10                       # chunks larger than every stage buffer


def test_crc_shift_levels():
    c = sc.crc_shift_levels()
    assert all(w is not None for w in c.want)
    check_against_oracles(c)
    assert sum(len(p) > 4 << 20 for p in c.payloads) <= 6


def _chunk_paths(c: sc.Corpus, override: int):
    """The ways a corpus's tasks are read when it is pushed into an empty ring and drained in windows of 4000."""
    tot = {}
    for lo in range(0, c.n, 4000):
        lens = [len(p) for p in c.payloads[lo:lo + 4000]]
        offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
        cap = sc.stage_cap(c.handler, len(lens), sum(lens), max(lens), override)
        for k, v in sc.read_paths(offs, lens, sc.tile_tasks(c.handler, len(lens)), cap).items():
            tot[k] = tot.get(k, 0) + v
    return tot


@pytest.mark.parametrize("handler", ["identity", "crc32", "vadd_f32", "json_sum"])
def test_mixed_windows(handler):
    c = sc.mixed_windows(handler)
    check_against_oracles(c)
    assert all(w is not None for w in c.want)
    for override in (0, 1024):
        p = _chunk_paths(c, override)
        assert p["2"] > 0 and p["3"] > 0, (override, p)
        assert override or p["1"] > 0
    assert max(len(x) for x in c.payloads) >= 1000 << 10


@pytest.mark.parametrize("handler", ["identity", "crc32", "vadd_f32", "json_sum"])
def test_exact_fit_tiles(handler):
    wins = sc.exact_fit_tiles(handler)
    assert len(wins) == (3 if handler == "vadd_f32" else 6)
    for w in wins:
        check_against_oracles(w.corpus)
        m = sc.RingModel(1 << 20)
        for k, n in enumerate(w.pushes):
            lo = sum(w.pushes[:k])
            assert m.push([len(p) for p in w.corpus.payloads[lo:lo + n]]) is not None
        offs, lens, _ = m.window(w.corpus.n)
        p = sc.read_paths(offs, lens, sc.tile_tasks(handler, w.corpus.n), 1024)
        staged = w.target <= 1024
        if w.scattered:
            assert offs[w.pushes[0]] == 256 * (-(-sum(lens[:w.pushes[0]]) // 256)) != sum(lens[:w.pushes[0]])
            assert p["4"] == (w.corpus.n if staged else 0) and p["4r"] == (0 if staged else 1), p
        else:
            assert p["1"] == (w.corpus.n if staged else 0) and p["fit"] == (w.target == 1024), p


def test_ring_model_matches_ring_place(script):  # noqa: F811
    rng = np.random.default_rng(9)
    for ring in (1024, 4096):
        ops, m, want = [], sc.RingModel(ring), []
        for _ in range(3000):
            if m.segs and rng.random() < 0.45:
                ops.append(POP)
                m.pop(len(m.segs[0][1]) - m.segs[0][2])
                want.append(0)
            else:
                b = int(rng.choice([0, int(rng.integers(1, ring // 2)), 256 * int(rng.integers(1, ring // 512 + 1))]))
                ops.append(PUSH(b))
                s = m.push([b] if b else [0])
                want.append(-1 if s is None else s)
        assert script(ring, ops) == want
