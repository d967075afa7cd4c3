"""Inputs of the function path's pickle codec tests (tests/test_pickle_on_host.py on a CPU, tests/test_gpu_function_full.py
on the device): cloudpickle blobs as `.map()` / `.remote()` send them, hand-assembled blobs for what the pickler never
writes itself (separate equal objects, memo references, FRAME placement), and a classifier of the documented declines."""
from __future__ import annotations

import base64
import json
import math
import os
import pickle
import pickletools
import random
import struct
from typing import Any, List, Optional

import cloudpickle

from beta9_b200 import synth
from oracle.pyoracle import funcloop

HANDLERS = ["identity", "crc32", "vadd_f32", "json_sum"]
HERE = os.path.dirname(os.path.abspath(__file__))
ALLOWED_OPS = {"PROTO", "FRAME", "EMPTY_DICT", "EMPTY_LIST", "EMPTY_TUPLE", "MARK", "TUPLE1", "TUPLE2", "TUPLE3", "TUPLE",
               "APPEND", "APPENDS", "SETITEM", "SETITEMS", "MEMOIZE", "BINGET", "LONG_BINGET", "SHORT_BINUNICODE",
               "BINUNICODE", "BINUNICODE8", "SHORT_BINBYTES", "BINBYTES", "BINBYTES8", "BININT1", "BININT2", "BININT", "LONG1",
               "BINFLOAT", "NONE", "NEWTRUE", "NEWFALSE", "STOP"}
MAX_NODES, MAX_MEMO, MAX_MARKS, MAX_DEPTH, MAX_MEMBERS, FRAME_TARGET = 2048, 1024, 32, 16, 64, 65536


# ---- hand-assembled blobs
def s_op(s: str) -> bytes:
    b = s.encode("utf-8", "surrogatepass")
    return (b"\x8c" + bytes([len(b)]) if len(b) < 256 else b"X" + struct.pack("<I", len(b))) + b


def framed(body: bytes) -> bytes:
    """PROTO 5 + one FRAME around `body` (which ends with STOP)."""
    return b"\x80\x05\x95" + struct.pack("<Q", len(body)) + body


def call_blob(arg_ops: bytes, kwargs_ops: bytes = b"}") -> bytes:
    """{"args": (<arg_ops>,), "kwargs": <kwargs_ops>} with the pickler's own layout around the argument."""
    return framed(b"}(" + s_op("args") + arg_ops + b"\x85" + s_op("kwargs") + kwargs_ops + b"u.")


def hand_built() -> List[bytes]:
    e = s_op("é")
    out = [
        call_blob(b"]\x94(" + e + e + b"e"),                       # two separate "é": one object after loading
        call_blob(b"]\x94(" + s_op("Ā") + s_op("Ā") + b"e"),      # "Ā": two objects
        call_blob(b"]\x94(" + s_op("ab") + s_op("ab") + b"e"),
        call_blob(b"]\x94(" + s_op("") + s_op("") + s_op("a") + s_op("a") + b"e"),
        call_blob(b"]\x94(C\x00C\x00C\x01xC\x01xe"),               # b"" collapses, b"x" does not
        call_blob(b"]\x94()))e"),                                  # () twice
        call_blob(b"]\x94(\x8c\x01a\x94h\x01h\x01e"),              # a memo reference to a str
        call_blob(b"]\x94(]\x94K\x01a h\x01e".replace(b" ", b"")),   # a shared list
        call_blob(b"]\x94\x94h\x01a"),                             # a cycle: the list appended to itself
        call_blob(b"K\x05", b"}\x94" + s_op("callback_url") + b"K\x01s"),
        call_blob(b"K\x05", b"}\x94" + s_op("callback_url") + b"K\x01" + s_op("callback_url") + b"K\x02u"),
        call_blob(b"K\x05", b"}\x94" + s_op("x") + b"K\x01s"),
        call_blob(b"K\x05", b"]"),                                 # falsy kwargs of another type
        call_blob(b"K\x05", b"K\x01"),                             # truthy kwargs of another type
        call_blob(b"\x8a\x09" + b"\x00" * 8 + b"\x01"),            # LONG1 of a non-minimal length
        call_blob(b"\x8a\x08" + b"\xff" * 8),                      # LONG1 -1
        call_blob(b"\x8a\x00"),                                    # LONG1 0
        call_blob(b"\x8a\x02\x00\x00"),
        call_blob(b"J\x05\x00\x00\x00"),                           # BININT for a small int
        call_blob(b"}\x94(K\x01K\x01G?\xf0\x00\x00\x00\x00\x00\x00K\x02u"),   # {1: 1, 1.0: 2}: equal keys
        call_blob(b"}\x94(G\x7f\xf8\x00\x00\x00\x00\x00\x00K\x01G\x7f\xf8\x00\x00\x00\x00\x00\x00K\x02u"),   # two NaN keys
        call_blob(b"}\x94(\x88K\x01K\x01K\x02u"),                  # {True: 1, 1: 2}
        call_blob(b"}\x94(G\x00\x00\x00\x00\x00\x00\x00\x00K\x01G\x80\x00\x00\x00\x00\x00\x00\x00K\x02u"),   # 0.0, -0.0
        call_blob(b"}\x94(C\x01aK\x01\x8c\x01aK\x02u"),            # b"a", "a": different keys
        call_blob(b"}\x94(\x8a\x09\x00\x00\x00\x00\x00\x00\x00\x00\x01K\x01G\x43\xf0\x00\x00\x00\x00\x00\x00K\x02u"),   # 2^64 twice
        b"\x80\x05" + b"}(" + s_op("args") + b"\x95\x02\x00\x00\x00\x00\x00\x00\x00K\x07\x85" + s_op("kwargs") + b"}u.",   # FRAME inside
        b"\x80\x05}(" + s_op("args") + b"K\x07\x85" + s_op("kwargs") + b"}u.",             # no frame at all
        call_blob(b"K\x05") + b"X",                                # data after STOP
        call_blob(b"\x8c\x02\xed\xa0"),                            # a lone surrogate: str, not for crc32
        call_blob(b"\x8c\x03\xed\xa0\x80"),
        call_blob(b"\x8c\x02\xc0\x80"),                            # overlong UTF-8
        framed(b"]."),                                             # payload not a dict
        framed(b"}(" + s_op("args") + b"K\x01K\x02\x86" + s_op("args") + b"K\x03\x85u."),   # "args" twice: the last wins
        framed(b"}(" + s_op("args") + s_op("ab") + b"u."),         # args a str
        framed(b"}(" + s_op("args") + b"]u."),                     # args empty
        framed(b"}."),
    ]
    return out


# ---- blobs the SDK sends
def nan_payload(bits: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


def plain_values() -> List[Any]:
    ints = [0, 1, 255, 256, 65535, 65536, 2**31 - 1, 2**31, -2**31, -2**31 - 1, 2**32, 2**63 - 1, 2**63, -2**63, -2**63 - 1,
            2**64, 10**30, -10**30, -1, -128, -129, -256, -257, -32768, -32769, 2**2039]
    floats = [0.0, -0.0, 1.5, math.inf, -math.inf, math.nan, nan_payload(0x7FF8000000000001), nan_payload(0xFFF0000000000123),
              5e-324, 1e308, 2.0**63, -2.0**63, 1e30]
    strs = ["", "a", "é", "Ā", "€", "\U0001f600", "\ud83d", "args", "kwargs", "callback_url", "x" * 255, "y" * 256, "z" * 70000]
    vals: List[Any] = ints + floats + strs + [None, True, False, b"", b"x", b"bytes" * 60, (), [], {}]
    vals += [[1], [1, 2], (1,), (1, 2), (1, 2, 3), (1, 2, 3, 4), {"a": 1}, {"a": 1, "b": [2, 3]}, [[1, 2]] * 3, ("t", ("u",))]
    vals += [list(range(n)) for n in (999, 1000, 1001, 2000)]
    vals += [[str(i) for i in range(300)], [s for s in ["é"] * 5], {str(i): i for i in range(64)}, {str(i): i for i in range(65)}]
    vals += [{1: "a", 2.5: "b", None: "c", True: "d", b"k": "e", "k": "f"}]
    shared = ["s" * 3]
    vals += [[shared, shared], [shared] * 300 + [str(i) for i in range(300)]]
    deep: Any = 1
    for _ in range(20):
        deep = [deep]
    vals += [deep]
    cyc: List[Any] = []
    cyc.append(cyc)
    vals += [cyc]
    # results at 3, 4 and 5 body bytes and at the 64 KiB frame target
    vals += [0, 256, (1,), "q" * 65527, "q" * 65528, "q" * 65529, "q" * 65530, b"r" * 65528, b"r" * 65530]
    return vals


def vadd_values() -> List[Any]:
    rng = random.Random(7)
    raw = [bytes(rng.randrange(256) for _ in range(8 * k)) for k in (0, 1, 2, 5, 16)]
    out: List[Any] = [base64.b64encode(r).decode() for r in raw] + [base64.b64encode(r) for r in raw]
    out += ["AAAA", "AAAAAAAA====", "AAAA=AAA", "é", b"\xff\xff\xff\xff", base64.b64encode(b"1234567").decode(), 5, None]
    return out


def json_sum_values() -> List[Any]:
    from tests.f64_corpus import sum_edge_payloads
    docs: List[Any] = []
    for p in sum_edge_payloads():
        try:
            a = json.loads(p)["args"][0]
        except Exception:
            continue
        docs.append(a)
    docs += [{"values": [1, 2.5, True]}, {"values": (1, 2)}, {"values": [2**63 - 1, 1]}, {"values": [2**64]}, {"values": [1.5, 2**64]},
             {"values": [1, None]}, {"values": [2**64, None]}, {"values": "ab"}, {"values": None}, {"values": []}, {"v": [1]},
             {"values": [1], "values2": 3}, [1, 2], {"values": [math.inf, -math.inf]}, {"values": [1e308, 1e308, -1e308]},
             {"values": [0.1] * 10}, {"values": [-0.0]}, {"values": [math.nan, 1]}]
    return docs


def sdk_blobs(n_docs: int = 200) -> List[bytes]:
    b = synth.function_docs_batch(n_docs)
    raw = b.payload.tobytes()
    blobs = [raw[int(b.offsets[i]):int(b.offsets[i + 1])] for i in range(b.n)]
    fb = synth.json_float_batch(n_docs)
    fraw = fb.payload.tobytes()
    blobs += [funcloop.frame_map_input(json.loads(fraw[int(fb.offsets[i]):int(fb.offsets[i + 1])])["args"][0]) for i in range(fb.n)]
    vb = synth.values_batch(n_docs)
    vraw = vb.payload.tobytes()
    blobs += [funcloop.frame_map_input(json.loads(vraw[int(vb.offsets[i]):int(vb.offsets[i + 1])])["args"][0]) for i in range(vb.n)]
    return blobs


def frame_one(v: Any) -> bytes:
    """one argument, as `.remote(v)` sends it (`.map` would unpack a list or tuple)"""
    return funcloop.frame_call(v)


def structured_blobs() -> List[bytes]:
    vals = plain_values() + vadd_values() + json_sum_values()
    blobs = [frame_one(v) for v in vals]
    blobs += [funcloop.frame_map_input(x) for x in [("a", "b"), [], (), "s", 5]]
    blobs += [funcloop.frame_call("s", callback_url="http://x"), funcloop.frame_call(5, callback_url="u"), funcloop.frame_call("s", k=1)]
    golden = []
    for name in ("ref_function_golden.json", "ref_function_full_golden.json"):
        golden += json.load(open(os.path.join(HERE, "golden", name)))["cases"]
    blobs += [base64.b64decode(c["args_pickle"]) for c in golden]
    blobs += hand_built() + sdk_blobs()
    return blobs


def mutations(blobs: List[bytes], n: int, seed: int = 11) -> List[bytes]:
    rng = random.Random(seed)
    small = [b for b in blobs if len(b) < 4096]
    out = []
    for _ in range(n):
        b = bytearray(rng.choice(small))
        k = rng.randrange(4)
        if k == 0:
            b = b[:rng.randrange(len(b) + 1)]
        elif k == 1:
            for _ in range(rng.randrange(1, 4)):
                if b:
                    b[rng.randrange(len(b))] = rng.randrange(256)
        elif k == 2 and b:
            i = rng.randrange(len(b))
            del b[i:i + rng.randrange(1, 4)]
        else:
            i = rng.randrange(len(b) + 1)
            b[i:i] = bytes([rng.choice(b"}]()\x85\x86\x87taseu\x94hjKMJ\x8aGN\x88\x89.")])
        out.append(bytes(b))
    return out


# ---- the documented declines (include/b9gpu.h, B9_TF_PICKLE)
def _depth(v: Any, d: int = 0) -> int:
    if isinstance(v, (list, tuple, dict)) and not (isinstance(v, tuple) and not v):
        items = list(v.items()) if isinstance(v, dict) else v
        inner = [x for kv in items for x in (kv if isinstance(v, dict) else (kv,))]
        return max([d + 1] + [_depth(x, d + 1) for x in inner])
    return d


def declined(blob: bytes, handler: str) -> Optional[str]:
    """Why the device may answer UNSUPPORTED for this blob, or None when it must answer."""
    try:
        ops = list(pickletools.genops(blob))
    except Exception:
        return "ill-formed stream"
    if any(op.name not in ALLOWED_OPS for op, _, _ in ops):
        return "opcode"
    if ops[-1][0].name != "STOP" or ops[-1][2] + 1 != len(blob):
        return "ill-formed stream"
    if ops[0][0].name != "PROTO" or ops[0][1] != 5:
        if any(op.name == "PROTO" and arg != 5 for op, arg, _ in ops):
            return "opcode"
    pushes = sum(1 for op, _, _ in ops if op.name not in ("PROTO", "FRAME", "MARK", "MEMOIZE", "STOP", "APPEND", "APPENDS", "SETITEM", "SETITEMS"))
    if pushes > MAX_NODES or sum(1 for op, _, _ in ops if op.name == "MEMOIZE") > MAX_MEMO:
        return "scratch"
    kids = sum(1 for op, _, _ in ops if op.name in ("APPEND", "APPENDS", "SETITEM", "SETITEMS", "TUPLE", "TUPLE1", "TUPLE2", "TUPLE3"))
    if kids > 256:
        return "scratch"
    try:
        payload = pickle.loads(blob)
    except Exception:
        return "ill-formed stream"
    if not isinstance(payload, dict):
        return None
    seen = set()

    def walk(v: Any) -> Optional[str]:
        if id(v) in seen:
            return "cycle" if isinstance(v, (list, dict)) and any(x is v for x in (v.values() if isinstance(v, dict) else v)) else None
        if isinstance(v, (list, tuple, dict)):
            seen.add(id(v))
        if isinstance(v, dict):
            if len(v) > MAX_MEMBERS:
                return "dict members"
            for k, x in v.items():
                if type(k) not in (str, bytes, int, bool, float, type(None)):
                    return "key type"
                r = walk(x)
                if r:
                    return r
        elif isinstance(v, (list, tuple)):
            for x in v:
                r = walk(x)
                if r:
                    return r
        return None
    try:
        r = walk(payload)
    except RecursionError:
        return "cycle"
    if r:
        return r
    args, kwargs = payload.get("args"), payload.get("kwargs")
    if args and not isinstance(args, (list, tuple)):
        return "args type"
    if kwargs and not isinstance(kwargs, dict):
        return None
    if not args or len(args) != 1 or any(k != "callback_url" for k in (kwargs or {})):
        return None
    x = args[0]
    if handler == "json_sum" and isinstance(x, dict) and "values" in x:
        vals = x["values"]
        if not isinstance(vals, (list, tuple)):
            return "values type"
        if any(v is None or isinstance(v, (str, bytes, list, tuple, dict)) for v in vals):
            return None
        acc, fl = 0, False
        for v in vals:
            if isinstance(v, float):
                fl = True
            elif not -2**63 <= v < 2**63 or (not fl and not -2**63 <= acc + v < 2**63):
                return "C long range"
            elif not fl:
                acc += v
    if handler == "identity":
        if _depth(x) > MAX_DEPTH:
            return "depth"
        if len(cloudpickle.dumps(x)) >= FRAME_TARGET:
            return "frame target"
        if _dup_keys(blob):
            return "equal keys"
    return None


class _DupKeys(pickle._Unpickler):
    """the pure-Python unpickler, noting a SETITEM(S) whose key the dict holds already"""
    dup = False
    dispatch = dict(pickle._Unpickler.dispatch)

    def _set(self, d, k, v):
        if k in d:
            self.dup = True
        d[k] = v

    def load_setitem(self):
        v = self.stack.pop()
        k = self.stack.pop()
        self._set(self.stack[-1], k, v)
    dispatch[pickle.SETITEM[0]] = load_setitem

    def load_setitems(self):
        items = self.pop_mark()
        for i in range(0, len(items), 2):
            self._set(self.stack[-1], items[i], items[i + 1])
    dispatch[pickle.SETITEMS[0]] = load_setitems


def _dup_keys(blob: bytes) -> bool:
    import io
    u = _DupKeys(io.BytesIO(blob))
    try:
        u.load()
    except Exception:
        return False
    return u.dup
