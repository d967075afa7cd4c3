"""The Python twins of the contract handlers (contract.cuh).

`expect(ops, rendering)` is `script`'s twin: it applies the rules include/b9gpu_handler.cuh states (the counting sink,
the settle rules, the writing sink and its reservation) to a script and says what the record must be: UNSUPPORTED, an
ERROR of one B9_EXC_* class, or the Python value the script builds. The tests turn that value into record bytes with the
runner's own rendering (run_task_loop, the endpoint oracle), never by hand. `describe` is `inspect`'s twin, written from
the value json.loads gave the runner; `inspect_keys` is `inspect_keys`'s."""
import binascii
import json
import math
import struct

TQ, ENDPOINT = 0, 1
UNSUPPORTED, ERROR, VALUE = "UNSUPPORTED", "ERROR", "VALUE"
EXC_CLASSES = {0x01: TypeError, 0x02: AttributeError, 0x04: UnicodeEncodeError, 0x08: KeyError, 0x10: ValueError,
               0x20: binascii.Error}
EXC_ALL = 0x3F
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1

# op codes
NONE, BOOL, INT, REAL, STR_BEGIN, CP, STR_END, RETURN, CP_WRITE, CP_COUNT = range(10)

PROBES = ["a", "values", "é", "€", "\U0001F600", "", 'a"b']
DEPTH = 3


def exception(bit):
    """an instance of the class B9_EXC_* `bit` names"""
    cls = EXC_CLASSES[bit]
    return cls("utf-8", "\udc80", 0, 1, "surrogates not allowed") if cls is UnicodeEncodeError else cls("raised by the script")


def halves(v):
    """a 64-bit argument as the op's two unsigned 32-bit halves"""
    u = v & 0xFFFFFFFFFFFFFFFF
    return [u >> 32, u & 0xFFFFFFFF]


def _s64(u):
    u &= 0xFFFFFFFFFFFFFFFF
    return u - (1 << 64) if u >> 63 else u


def _c_int(v):
    """(int)v of a long long v"""
    return ((v & 0xFFFFFFFF) ^ 0x80000000) - 0x80000000


def _float(bits):
    return struct.unpack("<d", struct.pack("<Q", bits & 0xFFFFFFFFFFFFFFFF))[0]


def _cp_ok(c):
    return c <= 0x10FFFF and not 0xD800 <= c <= 0xDFFF


def cp_len(c, rendering):
    """the bytes one code point takes in a string result: json.dumps with ensure_ascii, or as JSONResponse writes it"""
    if rendering == ENDPOINT:
        return len(json.dumps(chr(c), ensure_ascii=False).encode()) - 2
    return len(json.dumps(chr(c))) - 2


def parse(ops):
    """[(code, argument)] of a script up to its first RETURN, as the handler reads it op by op; None for a malformed
    script (the handler raises TypeError when it meets the malformed op). Raises Unsure for an int outside int64."""
    if type(ops) is not list:
        return None
    out = []
    for op in ops:
        if type(op) is not list or not 1 <= len(op) <= 3 or any(type(x) is not int for x in op):
            return None
        if any(not INT64_MIN <= x <= INT64_MAX for x in op):
            raise Unsure()
        if not 0 <= op[0] <= CP_COUNT:
            return None
        v = _s64(((op[1] & 0xFFFFFFFF) << 32) | (op[2] & 0xFFFFFFFF)) if len(op) == 3 else op[1] if len(op) == 2 else 0
        out.append((op[0], v))
        if op[0] == RETURN:
            break
    return out


def _count_pass(ops):
    """CountSink over the ops up to the first RETURN: (return value, kind, value, open)"""
    kind, val, open_ = None, None, False
    bad = "bad"

    def start(k):
        nonlocal kind, open_
        if kind is not None or open_:
            kind, open_ = bad, False
            return False
        kind = k
        return True

    for code, v in ops:
        if code == RETURN:
            return _c_int(v), kind, val, open_
        if code == NONE:
            start("none")
        elif code == BOOL:
            if start("bool"):
                val = v != 0
        elif code == INT:
            if start("int"):
                val = v
        elif code == REAL:
            if start("float"):
                val = v & 0xFFFFFFFFFFFFFFFF
        elif code == STR_BEGIN:
            if start("str"):
                open_, val = True, []
        elif code in (CP, CP_COUNT):
            if not open_:
                kind = bad
            elif not _cp_ok(v & 0xFFFFFFFF):
                kind, open_ = bad, False
            else:
                val.append(v & 0xFFFFFFFF)
        elif code == STR_END:
            if not open_:
                kind = bad
            open_ = False
    return 0, kind, val, open_


def _write_pass(ops, cap, rendering):
    """WriteSink with a reservation of `cap` bytes: the code points written, or None where the sink refuses, the string
    is not closed, or fewer bytes than `cap` were written"""
    n, ok, open_, done, cps = 0, True, False, False, []
    for code, v in ops:
        if code == RETURN:
            break
        c = v & 0xFFFFFFFF
        if code in (NONE, BOOL, INT, REAL):
            ok = False
        elif code == STR_BEGIN:
            if done or open_ or cap < 2:
                ok = False
            else:
                n, open_ = 1, True
        elif code in (CP, CP_WRITE):
            if not ok or not open_ or not _cp_ok(c):
                ok = False
            elif n + cp_len(c, rendering) + 1 > cap:        # never past the reservation, closing quote included
                ok = False
            else:
                n += cp_len(c, rendering)
                cps.append(c)
        elif code == STR_END:
            if not ok or not open_:
                ok = False
            else:
                n, open_, done = n + 1, False, True
    return "".join(map(chr, cps)) if ok and done and n == cap else None


def expect(ops, rendering):
    """(UNSUPPORTED, None), (ERROR, the B9_EXC_* bit) or (VALUE, the Python value) of `script(ops)` in `rendering`"""
    try:
        parsed = parse(ops)
    except Unsure:
        return UNSUPPORTED, None
    if parsed is None:
        return ERROR, 0x01
    ret, kind, val, open_ = _count_pass(parsed)
    if ret != 0:                                  # one B9_EXC_* bit raises that class; anything else is UNSUPPORTED
        return (ERROR, ret) if 0 < ret <= EXC_ALL and not ret & (ret - 1) else (UNSUPPORTED, None)
    if kind in (None, "bad") or open_:            # no value, a broken rule, a string left open
        return UNSUPPORTED, None
    if kind == "none":
        return VALUE, None
    if kind in ("bool", "int"):
        return VALUE, val
    if kind == "float":
        x = _float(val)
        if rendering == ENDPOINT and not math.isfinite(x):
            return UNSUPPORTED, None              # allow_nan=False
        return VALUE, x
    if rendering == TQ and not val:               # a falsy "" has no record bytes: no writing pass
        return VALUE, ""
    counted = 2 + sum(cp_len(c, rendering) for c in val)
    s = _write_pass(parsed, counted, rendering)
    return (UNSUPPORTED, None) if s is None else (VALUE, s)


def twin(rendering, signature=False):
    """script's Python twin for one rendering (signature: script_sig's): returns expect's value or raises its class, or
    Declined where the device must decline"""
    def script(ops, /):
        kind, x = expect(ops, rendering)
        if kind == ERROR:
            raise exception(x)
        if kind == UNSUPPORTED:
            raise Declined()
        return x

    def script_sig(ops, *rest):
        return script(ops)
    return script_sig if signature else script


class Declined(Exception):
    """the device must answer UNSUPPORTED"""


class Unsure(Exception):
    """number() cannot answer exactly: an int outside int64"""


# ---- inspect ------------------------------------------------------------------------------------------------------------
def _kind(v):
    if type(v) is str:
        return "S"
    if type(v) is bool:
        return "B"
    if type(v) is int:
        return "I"
    if type(v) is float:
        return "F"
    if v is None:
        return "N"
    return "L" if type(v) is list else "D"


def head(v):
    k = _kind(v)
    out = k + ("1" if k in "SLD" and len(v) == 0 else "0")
    if k in "BI":
        if not INT64_MIN <= v <= INT64_MAX:
            raise Unsure()
        out += "=i%d" % int(v)
    elif k == "F":
        out += "=f%x" % struct.unpack("<Q", struct.pack("<d", v))[0]
    elif k == "S":
        out += ":" + ".".join("%x" % ord(c) for c in v)
    return out


def describe(v, depth=0):
    """inspect's description of a value (contract.cuh: head, items, probe keys, DEPTH levels)"""
    out = head(v)
    if depth >= DEPTH:
        return out
    if type(v) is list:
        return out + "[" + ",".join(describe(x, depth + 1) for x in v) + "]"
    if type(v) is dict:
        return out + "{" + ",".join(describe(v[k], depth + 1) if k in v else "-" for k in PROBES) + "}"
    return out


def inspect(v, /):
    return describe(v)


def inspect_keys(d, *keys):
    def found(k):
        return describe(d[k]) if type(d) is dict and type(k) is str and k in d else "-"
    parts = []
    for k in keys:
        s = found(k)
        if type(k) is str and k in PROBES:
            s += "|" + found(k)
        parts.append(s)
    return ";".join(parts)
