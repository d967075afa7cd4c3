"""CPU checks of the retry policy (b9_set_retry_policy, include/b9gpu.h):

* the retry oracle's runner half (tests/retry_oracle.py) against the reference's own runner with a stub `retry_for`,
  frozen in tests/golden/ref_retry_golden.json by tests/golden/make_ref_retry_golden.py;
* the exception class the device's sequential path hands to the policy (an ERROR's TaskRec::value, compiled for the host by
  tests/host_shim/retry_shim.cpp) against the oracle's type(e), for every ERROR of the fuzz corpus, the float64 corpus,
  the TaskMessage mutants and a corpus written for each class: no device ERROR falls outside the six B9_EXC_* classes;
* the binding's mapping of `retry_for` classes to B9_EXC_* bits.
"""
import binascii
import ctypes as C
import json
import os
import subprocess

import pytest

from beta9_b200.device_queue import EXC_BITS, retry_mask
from oracle.pyoracle.handlers import HANDLERS as FUNCS
from oracle.pyoracle.loop import sdk_put_payload
from tests import f64_corpus
from tests.golden.make_ref_retry_golden import CLASSES, LETTER, corpus_wires
from tests.golden.make_ref_runner_golden import fuzz_payloads
from tests.retry_oracle import RETRY_LIMIT, call_handler, run_retry_loop

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_shim", "retry_shim.cpp")
SO = os.path.join(HERE, "host_shim", "libretry.so")
GXX = os.environ.get("CXX", "g++")
HANDLERS = {"identity": 0, "crc32": 1, "vadd_f32": 2, "json_sum": 3}
ST_ERROR, ST_UNSUPPORTED = 1, 4
KIND_PAYLOAD, KIND_HTTP, KIND_RECORD = 0, 1, 2


def _golden():
    return json.load(open(os.path.join(HERE, "golden", "ref_retry_golden.json")))


# ---------------------------------------------------------------------------------------------- 1. the oracle's runner half
@pytest.mark.parametrize("handler", list(HANDLERS))
def test_oracle_runner_half_equals_the_reference_with_each_retry_for_class(handler):
    ref = _golden()["handlers"][handler]
    wires = corpus_wires(handler)
    assert len(wires) == ref["n"] and len(wires) > 1000
    tasks = [json.loads(w) for w in wires]
    for name, cls in CLASSES.items():
        got = "".join(LETTER[call_handler(FUNCS[handler], t["args"], t["kwargs"], [cls])[0]] for t in tasks)
        assert got == ref["status"][name], name


@pytest.mark.parametrize("handler", list(HANDLERS))
def test_oracle_exception_class_is_the_one_the_reference_retries_on(handler):
    """A task the reference retries under retry_for = [c] raised exactly c (retry_on_errors is `type(e) is err`), and only
    for that one class; a task that completes is retried under none."""
    ref = _golden()["handlers"][handler]["status"]
    names = {cls: name for name, cls in CLASSES.items()}
    for i, w in enumerate(corpus_wires(handler)):
        t = json.loads(w)
        status, _, exc = call_handler(FUNCS[handler], t["args"], t["kwargs"], ())
        retried = {name for name in CLASSES if ref[name][i] == "R"}
        if status == "ERROR":
            assert retried == {names[exc]}, (w[:160], exc, retried)
        else:
            assert not retried and exc is None


def test_oracle_gateway_half_retries_up_to_max_retries_then_stops():
    ids = [bytes([i]) * 16 for i in range(3)]
    pl = [sdk_put_payload({}), sdk_put_payload({"values": [1, 2]}), sdk_put_payload({"values": [1]}, k=1)]
    got = [(a.task_id[0], a.status) for a in run_retry_loop(pl, ids, "json_sum", retry_for=[KeyError], max_retries=2)]
    assert got == [(0, "RETRY"), (1, "COMPLETE"), (2, "ERROR"), (0, "RETRY"), (0, RETRY_LIMIT)]
    got = [(a.task_id[0], a.status) for a in run_retry_loop(pl, ids, "json_sum", retry_for=[KeyError], max_retries=3, retries=[3, 0, 0])]
    assert got == [(0, RETRY_LIMIT), (1, "COMPLETE"), (2, "ERROR")]
    assert [a.status for a in run_retry_loop(pl, ids, "json_sum")] == ["ERROR", "COMPLETE", "ERROR"]


@pytest.mark.parametrize("handler", list(HANDLERS))
def test_retry_loop_without_a_policy_is_the_task_loop(handler):
    """With retry_for empty the retry loop answers every task exactly as oracle.pyoracle.loop.run_task_loop does (each
    task once, FIFO, REJECTED where the gateway refuses the push), over the fuzz payloads and the golden payloads, as SDK
    payloads and as HTTP bodies: the two loops share the push half's semantics."""
    from oracle.pyoracle import loop
    fz = json.load(open(os.path.join(HERE, "golden", "ref_fuzz_golden.json")))
    payloads, ids = fuzz_payloads(fz["n_payloads"], fz["seed"])
    golden = json.load(open(os.path.join(HERE, "golden", "hot_path_golden.json")))
    import base64
    gp = [base64.b64decode(c["payload"]) for cases in golden["groups"].values() for c in cases]
    payloads = list(payloads) + gp
    ids = list(ids) + _ids(len(gp), 3)
    for http in (False, True):
        want = loop.run_task_loop(payloads, ids, handler, http_body=http)
        got = run_retry_loop(payloads, ids, handler, http_body=[http] * len(payloads))
        assert [(a.task_id, a.status, a.result) for a in got] == [(w.task_id, w.status, w.result) for w in want]
        assert sum(a.status == "REJECTED" for a in got) > 0


# ---------------------------------------------------------------------------------------------- 2. the binding
def test_retry_for_maps_to_bits_by_class_identity():
    assert retry_mask(None) == 0 and retry_mask([]) == 0
    assert retry_mask(list(EXC_BITS)) == 0x3F
    assert retry_mask([ValueError]) == EXC_BITS[ValueError] != EXC_BITS[binascii.Error]
    assert retry_mask([binascii.Error]) == 0x20
    # subclasses and classes no device handler raises add nothing
    assert retry_mask([Exception, LookupError, UnicodeError, UnicodeDecodeError, RuntimeError, ZeroDivisionError]) == 0


# ---------------------------------------------------------------------------------------------- 3. the device's class
@pytest.fixture(scope="module")
def dev():
    csrc = os.path.join(os.path.dirname(HERE), "beta9_b200", "csrc")
    deps = [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".h"))]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max([os.path.getmtime(SRC)] + [os.path.getmtime(d) for d in deps]):
        r = subprocess.run([GXX, "-O2", "-std=c++17", "-shared", "-fPIC", "-o", SO, SRC], capture_output=True, text=True)
        if r.returncode:
            pytest.skip("no host C++ compiler for the shim: " + r.stderr[-300:])
    lib = C.CDLL(SO)
    lib.b9_retry_classify.argtypes = [C.c_char_p, C.c_uint32, C.c_int, C.c_char_p, C.c_int, C.POINTER(C.c_uint8), C.POINTER(C.c_uint8)]
    lib.b9_retry_classify.restype = None

    def run(b: bytes, kind: int, tid: bytes, handler: str):
        st, exc = C.c_uint8(0), C.c_uint8(0)
        lib.b9_retry_classify(b, len(b), kind, tid, HANDLERS[handler], C.byref(st), C.byref(exc))
        return int(st.value), int(exc.value)
    return run


def _check(dev, payloads, ids, handler, kind=KIND_PAYLOAD):
    """Every device ERROR carries the B9_EXC_* bit of the oracle's type(e), and the device answers ERROR exactly where
    the oracle does (UNSUPPORTED aside). Returns the number of ERRORs checked."""
    flags = [True] * len(payloads)
    want = run_retry_loop(payloads, ids, handler, http_body=flags if kind == KIND_HTTP else (),
                          task_msg=flags if kind == KIND_RECORD else ())
    assert len(want) == len(payloads)                                      # (no retry_for: one answer per task, FIFO)
    n = 0
    for p, tid, a in zip(payloads, ids, want):
        st, exc = dev(bytes(p), kind, tid, handler)
        if st == ST_ERROR:
            assert a.status == "ERROR" and exc == EXC_BITS[a.exc], (bytes(p)[:160], a.status, a.exc, exc)
            n += 1
        else:
            assert exc == 0, (bytes(p)[:160], st, exc)
            if st != ST_UNSUPPORTED:
                assert a.status != "ERROR", (bytes(p)[:160], st, a.exc)
    return n


def _ids(n, salt):
    return [bytes([salt, (i >> 16) & 255, (i >> 8) & 255, i & 255]) * 4 for i in range(n)]


@pytest.mark.parametrize("handler", list(HANDLERS))
def test_device_class_on_the_fuzz_corpus(dev, handler):
    fz = json.load(open(os.path.join(HERE, "golden", "ref_fuzz_golden.json")))
    payloads, ids = fuzz_payloads(fz["n_payloads"], fz["seed"])
    assert _check(dev, payloads, ids, handler) > 100


@pytest.mark.parametrize("handler", ["identity", "json_sum"])
def test_device_class_on_the_float64_corpus(dev, handler):
    items = f64_corpus.sum_edge_payloads() + f64_corpus.value_edge_payloads()
    payloads = [p for p, _ in items]
    _check(dev, payloads, _ids(len(payloads), 7), handler)


# one corpus per class, with JSON values of every kind around them: SDK payloads, the same as HTTP bodies
CLASS_ARGS = {
    "identity": [[], ["a", "b"], [1, 2, 3], ["x"]],
    "crc32": [[1], [None], [[1]], [{"a": 1}], [True], [0.5], ["ok"], ["café"], ["\ud83d"], []],
    "vadd_f32": [[1], [None], [["QUFB"]], ["AAAA"], ["AAAAAAAAAAA="], ["AAAAAAAAAAAAAAAAAAAAAA=="], ["A"], ["AAA*"], ["AA=A"],
                 ["café"], ["éAAA"], ["AAAAé"], ["\x7fAAA"], ["QUFB\n"], [""], ["AAAAAAAAAAA"], ["===="]],
    "json_sum": [[{}], [{"v": 1}], [{"values": 3}], [{"values": None}], [{"values": "ab"}], [{"values": ""}],
                 [{"values": {"k": 1}}], [{"values": {}}], [{"values": [1, "x"]}], [{"values": [1, None]}],
                 [{"values": [[1]]}], [{"values": [1, 2.5]}], [[1, 2]], ["s"], [3], [None], [True]],
}


def _class_corpus(handler):
    out = []
    for args in CLASS_ARGS[handler]:
        out.append(sdk_put_payload(*args))
        out.append(sdk_put_payload(*args, extra=1))                       # keyword arguments: TypeError
    return out


@pytest.mark.parametrize("handler", list(HANDLERS))
def test_device_class_on_the_class_corpus(dev, handler):
    payloads = _class_corpus(handler)
    assert _check(dev, payloads, _ids(len(payloads), 9), handler) >= len(CLASS_ARGS[handler])
    bodies = [json.dumps({"args": a}).encode() for a in CLASS_ARGS[handler]] + [json.dumps(a[0]).encode() for a in CLASS_ARGS[handler] if a and isinstance(a[0], dict)]
    _check(dev, bodies, _ids(len(bodies), 10), handler, KIND_HTTP)


def test_device_raises_every_class_but_unicode_encode_error(dev):
    """Each class appears in the corpora above; UnicodeEncodeError cannot: a lone surrogate never reaches the handler
    (Go's decoder turns it into U+FFFD, and a TaskMessage record holding one is declined)."""
    seen = set()
    for handler in HANDLERS:
        for i, p in enumerate(_class_corpus(handler)):
            st, exc = dev(p, KIND_PAYLOAD, bytes(16), handler)
            if st == ST_ERROR:
                seen.add(exc)
    assert seen == set(EXC_BITS.values()) - {EXC_BITS[UnicodeEncodeError]}


@pytest.mark.parametrize("handler", list(HANDLERS))
def test_device_class_on_the_task_msg_mutants(dev, handler):
    from tests.test_task_msg_on_host import MUTANTS, TID
    answered = [rec for rec, want in MUTANTS.values() if want == "answer"]
    _check(dev, answered, [TID] * len(answered), handler, KIND_RECORD)
    for rec, want in MUTANTS.values():
        if want == "decline":
            assert dev(rec, KIND_RECORD, TID, handler) == (ST_UNSUPPORTED, 0)


@pytest.mark.parametrize("handler", list(HANDLERS))
def test_device_class_on_records_of_the_class_corpus(dev, handler):
    """The class corpus as the TaskMessage records Go writes for it (B9_TF_TASK_MSG)."""
    from oracle.pyoracle import loop
    payloads = _class_corpus(handler)
    ids = _ids(len(payloads), 11)
    live = loop.run_task_loop(payloads, ids, "identity", keep_wire=True)
    recs = [(w.wire, w.task_id) for w in live if w.wire is not None]
    assert _check(dev, [r for r, _ in recs], [t for _, t in recs], handler, KIND_RECORD) > 0
