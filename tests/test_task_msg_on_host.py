"""B9_TF_TASK_MSG on a CPU: the runner's half of the loop over TaskMessage records.

* the record oracle (tests/task_msg_oracle.py) against the reference runner's own answers for every golden wire record,
  and against the full oracle loop on the 1200 seeded fuzz payloads;
* the device's record path (task_msg.cuh + handler_phase_a, compiled for the host by tests/host_shim/task_msg_shim.cpp)
  against that oracle: the same status and bytes, and no decline of a Go-written record whose payload the payload path
  answers;
* named mutants and seeded byte mutations: the device's status is the oracle's or UNSUPPORTED, never a wrong answer."""
import base64
import ctypes as C
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

from oracle.pyoracle import loop
from oracle.pyoracle.wire import format_uuid
from tests.task_msg_oracle import NOT_RUN, run_records

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_shim", "task_msg_shim.cpp")
SO = os.path.join(HERE, "host_shim", "libtaskmsg.so")
GXX = os.environ.get("CXX", "g++")
HANDLERS = {"identity": 0, "crc32": 1, "vadd_f32": 2, "json_sum": 3}
CODE = {"COMPLETE": 0, "ERROR": 1, "RETRY": 2, NOT_RUN: 4}
UNSUPPORTED = 4


@pytest.fixture(scope="module")
def dev():
    csrc = os.path.join(os.path.dirname(HERE), "beta9_b200", "csrc")
    deps = [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".h"))]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max([os.path.getmtime(SRC)] + [os.path.getmtime(d) for d in deps]):
        r = subprocess.run([GXX, "-O2", "-std=c++17", "-shared", "-fPIC", "-o", SO, SRC], capture_output=True, text=True)
        if r.returncode:
            pytest.skip("no host C++ compiler for the shim: " + r.stderr[-300:])
    lib = C.CDLL(SO)
    lib.b9_tm_run.argtypes = [C.c_char_p, C.c_uint32, C.c_int, C.c_char_p, C.c_int, C.POINTER(C.c_uint8), C.POINTER(C.c_uint8),
                              C.c_char_p, C.c_uint32]
    lib.b9_tm_run.restype = C.c_long
    lib.b9_tm_utf8_surrogatepass.argtypes = [C.c_char_p, C.c_uint32]

    def run(b: bytes, record: bool, tid: bytes, handler: str):
        st, has = C.c_uint8(0), C.c_uint8(0)
        buf = C.create_string_buffer(8 * len(b) + 64)
        n = lib.b9_tm_run(b, len(b), 1 if record else 0, tid, HANDLERS[handler], C.byref(st), C.byref(has), buf, len(buf))
        assert n >= 0
        return int(st.value), (buf.raw[:n] if has.value else None)
    run.utf8 = lambda b: bool(lib.b9_tm_utf8_surrogatepass(b, len(b)))
    return run


def _golden():
    hot = json.load(open(os.path.join(HERE, "golden", "hot_path_golden.json")))
    ref = json.load(open(os.path.join(HERE, "golden", "ref_runner_golden.json")))
    return hot, ref


def golden_records():
    """(group, index, payload, task id, record) of every golden case that became a task"""
    hot, _ = _golden()
    out = []
    for g, cases in hot["groups"].items():
        for i, c in enumerate(cases):
            if c["wire"] is not None:
                out.append((g, i, base64.b64decode(c["payload"]), bytes.fromhex(c["task_id"]), base64.b64decode(c["wire"])))
    return out


def fuzz_records():
    from tests.golden.make_ref_runner_golden import fuzz_payloads
    ref = json.load(open(os.path.join(HERE, "golden", "ref_fuzz_golden.json")))
    payloads, ids = fuzz_payloads(ref["n_payloads"], ref["seed"])
    live = loop.run_task_loop(payloads, ids, "identity", keep_wire=True)
    keep = [i for i, w in enumerate(live) if w.wire is not None]
    return [payloads[i] for i in keep], [ids[i] for i in keep], [live[i].wire for i in keep], ref


# ---------------------------------------------------------------------------------------------- 1. the record oracle
@pytest.mark.parametrize("handler", list(HANDLERS))
def test_record_oracle_equals_the_reference_runner(handler):
    _, ref = _golden()
    recs = golden_records()
    assert len(recs) >= 150
    got = run_records([r[4] for r in recs], [r[3] for r in recs], handler)
    for (g, i, _, _, wire), w in zip(recs, got):
        r_status, r_result, r_task_id = ref["groups"][g][str(i)][handler]
        assert w.status == r_status, (g, i, wire[:120])
        assert w.result == (None if r_result is None else base64.b64decode(r_result)), (g, i)
        assert json.loads(wire)["task_id"] == r_task_id


@pytest.mark.parametrize("handler", list(HANDLERS))
def test_record_oracle_equals_the_task_loop_on_the_fuzz_payloads(handler):
    payloads, ids, wires, ref = fuzz_records()
    assert len(wires) == ref["handlers"][handler]["n_wires"]
    assert hashlib.sha256(b"".join(wires)).hexdigest() == ref["handlers"][handler]["wire_sha256"]
    full = [w for w in loop.run_task_loop(payloads, ids, handler) if w.status != loop.REJECTED]
    half = run_records(wires, ids, handler)
    assert [(w.status, w.result) for w in half] == [(w.status, w.result) for w in full]


# ---------------------------------------------------------------------------------------------- 2. the device's record path
# Go-written records the device declines although the payload path answers the payload: none.
DECLINE_EXCEPTIONS = {}


def _check_go_records(dev, payloads, ids, wires, handler):
    want = run_records(wires, ids, handler)
    declined = []
    for p, tid, wire, w in zip(payloads, ids, wires, want):
        st, res = dev(wire, True, tid, handler)
        if st == UNSUPPORTED:
            assert res is None
            p_st, _ = dev(p, False, tid, handler)
            if p_st != UNSUPPORTED:
                declined.append(wire)
            continue
        assert w.status != NOT_RUN, wire
        assert st == CODE[w.status], (wire[:160], st, w.status)
        assert res == w.result, (wire[:160], res, w.result)
    unexplained = [d for d in declined if d not in DECLINE_EXCEPTIONS]
    assert not unexplained, unexplained[:3]


@pytest.mark.parametrize("handler", list(HANDLERS))
def test_device_record_path_on_the_golden_records(dev, handler):
    recs = golden_records()
    _check_go_records(dev, [r[2] for r in recs], [r[3] for r in recs], [r[4] for r in recs], handler)


@pytest.mark.parametrize("handler", list(HANDLERS))
def test_device_record_path_on_the_fuzz_records(dev, handler):
    payloads, ids, wires, _ = fuzz_records()
    _check_go_records(dev, payloads, ids, wires, handler)


def test_device_record_path_on_generated_batches(dev):
    from beta9_b200 import synth
    for batch, handlers in ((synth.values_batch(1500, seed=31), ["identity", "json_sum"]),
                            (synth.json_float_batch(300, seed=32), ["json_sum", "identity"]),
                            (synth.strings_batch(1500, 64, adversarial_frac=0.2, seed=33), ["identity", "crc32"]),
                            (synth.vadd_batch(200, seed=34), ["vadd_f32"])):
        payloads = batch.tasks()
        ids = [bytes(batch.task_ids[i]) for i in range(batch.n)]
        live = loop.run_task_loop(payloads, ids, "identity", keep_wire=True)
        keep = [i for i, w in enumerate(live) if w.wire is not None]
        for h in handlers:
            _check_go_records(dev, [payloads[i] for i in keep], [ids[i] for i in keep], [live[i].wire for i in keep], h)


def test_surrogatepass_utf8_agrees_with_python(dev):
    rng = np.random.default_rng(5)
    samples = [b"", b"abc", "é€😀".encode(), b"\xed\xa0\x80", b"\xed\xbf\xbf", b"\xc0\x80", b"\xf4\x90\x80\x80", b"\xe0\x80\x80", b"\xff"]
    samples += [bytes(rng.integers(0, 256, int(rng.integers(1, 8)), dtype=np.uint8)) for _ in range(20000)]
    for b in samples:
        try:
            b.decode("utf-8", "surrogatepass")
            ok = True
        except UnicodeDecodeError:
            ok = False
        assert dev.utf8(b) == ok, b


# ---------------------------------------------------------------------------------------------- 3. mutants
TID = bytes(range(0x10, 0x20))
TID_TEXT = format_uuid(TID)


def record(args: bytes = b'["hello"]', kwargs: bytes = b"{}", task_id: bytes = None, head: bytes = b"", tail: bytes = b"") -> bytes:
    tid = b'"' + TID_TEXT.encode() + b'"' if task_id is None else task_id
    return (head + b'{"task_id":' + tid + b',"workspace_name":"ws","stub_id":"s-1","executor":"taskqueue","args":' + args
            + b',"kwargs":' + kwargs + b',"policy":{"max_retries":3,"timeout":3600,"expires":"2026-10-15T12:00:00.5Z","ttl":7200},'
            b'"retries":0,"timestamp":1789970992}' + tail)


BASE = record()
# name -> (record, whether the device may answer it: "answer" = must equal the oracle, "decline" = must be UNSUPPORTED)
MUTANTS = {
    "go_record": (BASE, "answer"),
    "whitespace": (BASE.replace(b'"args":', b'"args" :  ').replace(b",", b", "), "answer"),
    "whitespace_around": (b" \n" + BASE + b"\t ", "answer"),
    "keys_reordered_top": (b'{"args":["hello"],"kwargs":{},"task_id":"' + TID_TEXT.encode() + b'","retries":0}', "answer"),
    "keys_reordered_in_args": (record(b'[{"b": 1, "a": 2}]'), "decline"),
    "keys_sorted_in_args": (record(b'[{"a": 2, "b": 1}]'), "answer"),
    "duplicate_args": (BASE.replace(b'"kwargs":{}', b'"kwargs":{},"args":["x"]'), "decline"),
    "duplicate_task_id": (BASE.replace(b'"kwargs":{}', b'"kwargs":{},"task_id":"' + TID_TEXT.encode() + b'"'), "decline"),
    "duplicate_key_in_args": (record(b'[{"a": 1, "a": 2}]'), "decline"),
    "Args": (BASE.replace(b'"args"', b'"Args"'), "decline"),
    "escaped_args_key": (BASE.replace(b'"args"', b'"\\u0061rgs"'), "decline"),
    "float_1.0": (record(b"[1.0]"), "decline"),
    "float_1E2": (record(b"[1E2]"), "decline"),
    "float_-0.0": (record(b"[-0.0]"), "decline"),
    "float_1e400": (record(b"[1e400]"), "decline"),
    "NaN": (record(b"[NaN]"), "decline"),
    "Infinity": (record(b"[Infinity]"), "decline"),
    "-Infinity_elsewhere": (BASE.replace(b'"retries":0', b'"retries":-Infinity'), "decline"),
    "int_1": (record(b"[1]"), "answer"),
    "int_-0": (record(b"[-0]"), "answer"),
    "float_0.5": (record(b"[0.5]"), "answer"),
    "float_1e+21": (record(b"[1e+21]"), "answer"),
    "lone_surrogate": (record(b'["\\ud83d"]'), "decline"),
    "surrogate_pair": (record(b'["\\ud83d\\ude00"]'), "answer"),
    "encoded_surrogate": (record(b'["\xed\xa0\x80"]'), "decline"),
    "invalid_utf8": (record(b'["\xff"]'), "decline"),
    "invalid_utf8_elsewhere": (BASE.replace(b'"ws"', b'"w\xc3"'), "decline"),
    "utf8_bom": (b"\xef\xbb\xbf" + BASE, "decline"),
    "leading_nul": (b"\x00" + BASE, "decline"),
    "args_string": (record(b'"abc"'), "decline"),
    "args_object": (record(b'{"a": 1}'), "decline"),
    "args_null": (record(b"null"), "answer"),
    "kwargs_list": (record(kwargs=b"[1]"), "decline"),
    "kwargs_null": (record(kwargs=b"null"), "answer"),
    "kwargs_nonempty": (record(kwargs=b'{"x": 1}'), "answer"),
    "task_id_upper": (record(task_id=b'"' + TID_TEXT.upper().encode() + b'"'), "decline"),
    "task_id_other": (record(task_id=b'"' + format_uuid(bytes(16)).encode() + b'"'), "decline"),
    "task_id_number": (record(task_id=b"7"), "decline"),
    "trailing_x": (BASE + b"x", "decline"),
    "raw_control": (record(b'["a\x01b"]'), "decline"),
    "raw_tab": (record(b'["a\tb"]'), "decline"),
    "lt_escape": (record(b'["\\u003cb\\u003e"]'), "answer"),
    "raw_lt": (record(b'["<b>"]'), "answer"),
    "raw_e_acute": (record('["é"]'.encode()), "answer"),
    "two_args": (record(b'["a", "b"]'), "answer"),
    "nested": (record(b'[[1, {"k": [true, null, "x"]}]]'), "answer"),
    "missing_kwargs": (BASE.replace(b'"kwargs":{},', b""), "decline"),
    "empty_object": (b"{}", "decline"),
    "not_an_object": (b'["hello"]', "decline"),
    "huge_int_elsewhere": (BASE.replace(b'"retries":0', b'"retries":' + b"9" * 5000), "decline"),
}


@pytest.mark.parametrize("name", list(MUTANTS))
@pytest.mark.parametrize("handler", list(HANDLERS))
def test_named_mutants(dev, name, handler):
    rec, want = MUTANTS[name]
    o = run_records([rec], [TID], handler)[0]
    st, res = dev(rec, True, TID, handler)
    if want == "decline":
        assert st == UNSUPPORTED and res is None, (name, st, res, o.status)
    else:
        assert o.status != NOT_RUN and st == CODE[o.status] and res == o.result, (name, st, res, o.status, o.result)


def test_seeded_byte_mutations(dev):
    """tens of thousands of mutated records: the device's answer is the oracle's or UNSUPPORTED"""
    rng = np.random.default_rng(20261015)
    from beta9_b200 import synth
    seeds = [MUTANTS[k][0] for k in MUTANTS if MUTANTS[k][1] == "answer"]
    seed_ids = [TID] * len(seeds)
    vb = synth.values_batch(300, seed=41)
    live = loop.run_task_loop(vb.tasks(), [bytes(vb.task_ids[i]) for i in range(vb.n)], "identity", keep_wire=True)
    seeds += [w.wire for w in live if w.wire is not None]
    seed_ids += [w.task_id for w in live if w.wire is not None]
    alphabet = list(b'{}[],:" 0159e.-+Etrun\\lfa') + [0x00, 0x1F, 0x7F, 0xC3, 0xA9, 0xED, 0xA0, 0xFF]
    answered = checked = 0
    for n in range(30000):
        k = int(rng.integers(0, len(seeds)))
        m = bytearray(seeds[k])
        for _ in range(int(rng.integers(1, 3))):
            pos = int(rng.integers(0, len(m)))
            op = int(rng.integers(0, 3))
            ch = int(rng.choice(alphabet))
            if op == 0: m[pos] = ch
            elif op == 1: del m[pos]
            else: m[pos:pos] = bytes([ch])
        m = bytes(m)
        handler = list(HANDLERS)[n % 4]
        o = run_records([m], [seed_ids[k]], handler)[0]
        st, res = dev(m, True, seed_ids[k], handler)
        checked += 1
        if st == UNSUPPORTED:
            assert res is None
            continue
        answered += 1
        assert o.status != NOT_RUN, m
        assert st == CODE[o.status] and res == o.result, (handler, m[:200], st, res, o.status, o.result)
    assert checked == 30000 and answered > 3000, answered
