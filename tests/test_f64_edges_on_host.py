"""The shared float64 corpora (tests/f64_corpus.py) on a CPU: the one-number restatements against the oracle's task
loop, and the json_sum / identity edge corpora through the device's sequential path compiled for the host
(tests/host_shim/host_parse.cpp) against the oracle's task loop. With these pinned here, tests/test_gpu_f64.py can
check millions of device tasks against the restatements, and a disagreement there points at the device build."""
import numpy as np

from oracle.pyoracle import loop
from tests.f64_corpus import (_literals, _patterns, identity_of_literal, json_sum_of_literal, literal_may_decline,
                              sum_edge_payloads, value_edge_payloads)
from tests.test_device_parser_on_host import parser  # noqa: F401  (the host-compiled parser + handlers)

HANDLERS = {"identity": 0, "json_sum": 3}
CODE = {"COMPLETE": 0, "ERROR": 1, "RETRY": 2, "REJECTED": 3}


def _ids(n):
    return [i.to_bytes(4, "little") * 4 for i in range(n)]


def _sample_literals():
    lits = _literals()
    rng = np.random.default_rng(31)
    pick = [lits[int(i)] for i in rng.choice(len(lits), size=20_000, replace=False)]
    xs = _patterns(3000, 32).view(np.float64).tolist()
    return pick + [repr(x) for x in xs] + ["%.17g" % x for x in xs] + ["1e400", "-1e309", "1e-400", "-0", "0e0", "-0.0e-5"]


def test_identity_restatement_against_the_task_loop():
    lits = _sample_literals()
    want = loop.run_task_loop([b'{"args": [' + s.encode() + b'], "kwargs": {}}' for s in lits], _ids(len(lits)), "identity")
    for s, w in zip(lits, want):
        assert identity_of_literal(s) == (CODE[w.status], w.result), (s, w)


def test_json_sum_restatement_against_the_task_loop():
    lits = _sample_literals() + ["9223372036854775807", "9223372036854774784", "-9223372036854775808", "1e19", "1e20", "-1e20"]
    want = loop.run_task_loop([b'{"args": [{"values": [' + s.encode() + b']}], "kwargs": {}}' for s in lits], _ids(len(lits)),
                              "json_sum")
    declinable = 0
    for s, w in zip(lits, want):
        st, res, may_decline = json_sum_of_literal(s)
        assert (st, res) == (CODE[w.status], w.result), (s, w)
        declinable += may_decline and not literal_may_decline(s)
    assert declinable >= 4                                   # the C long bound is exercised, not only the digit count


def _run_corpus(parser, corpus, handler):
    payloads = [p for p, _ in corpus]
    want = loop.run_task_loop(payloads, _ids(len(payloads)), handler)
    declined = 0
    for (p, may_decline), w in zip(corpus, want):
        st, res = parser.run(p, False, HANDLERS[handler])
        if st == 4:
            assert may_decline, (p[:200], w)
            declined += 1
            continue
        assert (st, res) == (CODE[w.status], w.result), (p[:200], st, (res or b"")[:200], w.status, (w.result or b"")[:200])
    return declined


def test_sum_edge_corpus_on_host(parser):
    corpus = sum_edge_payloads()
    declined = _run_corpus(parser, corpus, "json_sum")
    assert declined == sum(d for _, d in corpus)             # exactly the C long cases
    statuses = [st for st, _ in (parser.run(p, False, 3) for p, _ in corpus)]
    assert statuses.count(1) >= 5 and statuses.count(3) >= 2


def test_llong_min_total_on_host(parser):
    p = b'{"args": [{"values": [-9000000000000000000, -220000000000000000, -3372036854775808]}], "kwargs": {}}'
    assert parser.run(p, False, 3) == (0, b"-9223372036854775808")
    assert parser.run(p.replace(b"-", b""), False, 3) == (4, None)      # 2^63: beyond a C long
    p = b'{"args": [{"values": [9000000000000000000, 220000000000000000, 3372036854775807]}], "kwargs": {}}'
    assert parser.run(p, False, 3) == (0, b"9223372036854775807")


def test_value_edge_corpus_on_host(parser):
    corpus = value_edge_payloads()
    declined = _run_corpus(parser, corpus, "identity")
    assert declined >= 19                                    # depth 17 / 18 (12 + 1) and 65 / 100 members (6)
