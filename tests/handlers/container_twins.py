"""The Python twin of the container script handler (containers.cuh).

`expect(ops, rest, rendering)` applies the rules include/b9gpu_handler.cuh states for lists, dicts and value() (and
contract_twins' for scalars and strings) to a script: both sinks' rule checks, the depth and member limits, duplicate
keys, the two passes' byte counts. It says what the record must be: UNSUPPORTED, an ERROR of one B9_EXC_* class, or
the Python value the script builds. The tests turn that value into record bytes with the runner's own rendering
(run_task_loop, the endpoint oracle), so the device's bytes are checked against CPython's json."""
import json
import math

from tests.handlers import contract_twins as CT
from tests.handlers.contract_twins import ENDPOINT, ERROR, TQ, UNSUPPORTED, VALUE, Declined, Unsure  # noqa: F401

NONE, BOOL, INT, REAL, STR_BEGIN, CP, STR_END, RETURN, CP_WRITE, CP_COUNT = range(10)
LIST_BEGIN, LIST_END, DICT_BEGIN, DICT_END, VALUE_OF = range(10, 15)
MAX_DEPTH, MAX_MEMBERS = 16, 64


def parse(ops, nrest):
    """[(code, argument)] up to the first RETURN; None for a malformed script (TypeError); raises Unsure for an int
    outside int64"""
    if type(ops) is not list:
        return None
    out = []
    for op in ops:
        if type(op) is not list or not 1 <= len(op) <= 3 or any(type(x) is not int for x in op):
            return None
        if any(not CT.INT64_MIN <= x <= CT.INT64_MAX for x in op):
            raise Unsure()
        if not 0 <= op[0] <= VALUE_OF:
            return None
        v = CT._s64(((op[1] & 0xFFFFFFFF) << 32) | (op[2] & 0xFFFFFFFF)) if len(op) == 3 else op[1] if len(op) == 2 else 0
        if op[0] == VALUE_OF and not 0 <= v < nrest:
            return None
        out.append((op[0], v))
        if op[0] == RETURN:
            break
    return out


def identity_declines(v, depth=0):
    """py_value_json / ep_value_json decline: a non-empty container nested past 16, a dict of more than 64 members"""
    if type(v) in (list, dict) and v:
        if depth == MAX_DEPTH or (type(v) is dict and len(v) > MAX_MEMBERS):
            return True
        return any(identity_declines(x, depth + 1) for x in (v.values() if type(v) is dict else v))
    return False


class _Bad(Exception):
    """a broken rule: the sink's value is VK_BAD"""


class _Dict:
    """a built dict: its members in the order written, duplicates kept"""
    def __init__(self):
        self.items, self.key = [], None


_UNSET, _PENDING = object(), object()


def run_pass(ops, rest, rendering, writing):
    """One sink over the ops: (return value, the built value, its top-level kind: "scalar", "str", "container" or
    "value"); the built value is _Bad where a rule broke. The writing pass (writing=True) also checks each built dict's
    keys; a top-level number, bool or None belongs to the counting pass alone."""
    top, kind, stack, string, is_key, bad = _UNSET, None, [], None, False, False

    def put(x, k):
        nonlocal top, kind
        if not stack:
            if top is not _UNSET:
                raise _Bad()                               # a second top-level value
            top, kind = x, k
            return
        c = stack[-1]
        if type(c) is list:
            c.append(x)
        elif c.key is None:
            raise _Bad()                                    # a non-string key
        else:
            c.items.append((c.key, x))
            c.key = None

    ret = 0
    for code, v in ops:
        if code == RETURN:
            ret = CT._c_int(v)
            break
        if bad:
            continue
        try:
            if code not in (CP, CP_WRITE, CP_COUNT, STR_END) and string is not None:
                raise _Bad()                               # a value or container call inside an open string
            if code in (NONE, BOOL, INT, REAL):
                x = None if code == NONE else v != 0 if code == BOOL else v if code == INT else CT._float(v)
                if stack and rendering == ENDPOINT and code == REAL and not math.isfinite(x):
                    raise _Bad()
                if writing and not stack:
                    raise _Bad()
                put(x, "scalar")
            elif code == STR_BEGIN:
                is_key = bool(stack) and type(stack[-1]) is _Dict and stack[-1].key is None
                if not is_key:
                    put(_PENDING, "str")
                string = []
            elif code == CP or code == (CP_WRITE if writing else CP_COUNT):
                if string is None or not CT._cp_ok(v & 0xFFFFFFFF):
                    raise _Bad()
                string.append(v & 0xFFFFFFFF)
            elif code == STR_END:
                if string is None:
                    raise _Bad()
                s, string = "".join(map(chr, string)), None
                if is_key:
                    stack[-1].key = s
                elif not stack:
                    top = s
                elif type(stack[-1]) is list:
                    stack[-1][-1] = s
                else:
                    stack[-1].items[-1] = (stack[-1].items[-1][0], s)
            elif code in (LIST_BEGIN, DICT_BEGIN):
                c = [] if code == LIST_BEGIN else _Dict()
                put(c, "container")
                if len(stack) == MAX_DEPTH:
                    raise _Bad()
                stack.append(c)
            elif code in (LIST_END, DICT_END):
                if not stack or (type(stack[-1]) is list) != (code == LIST_END):
                    raise _Bad()
                c = stack.pop()
                if type(c) is _Dict:
                    if c.key is not None:
                        raise _Bad()                       # a key with no value
                    keys = [k for k, _ in c.items]
                    if writing and (len(keys) > MAX_MEMBERS or len(set(keys)) != len(keys)):
                        raise _Bad()
            elif code == VALUE_OF:
                put(rest[v], "value")
                if identity_declines(rest[v]):
                    raise _Bad()
        except _Bad:
            bad = True
    if top is _UNSET or string is not None or stack:
        bad = True                                         # no value, a string or container left open
    return ret, _Bad if bad else top, kind


def _py(x):
    """the Python value of what a pass built"""
    if type(x) is _Dict:
        return {k: _py(v) for k, v in x.items}
    if type(x) is list:
        return [_py(v) for v in x]
    return x


def _len(x, rendering):
    """the bytes of the record of x (built dicts keep their members in order, duplicates included)"""
    if type(x) is _Dict:
        sep = ", " if rendering == TQ else ","
        col = ": " if rendering == TQ else ":"
        return 2 + sum(_len(k, rendering) + len(col) + _len(v, rendering) for k, v in x.items) + len(sep) * max(len(x.items) - 1, 0)
    if type(x) is list:
        sep = ", " if rendering == TQ else ","
        return 2 + sum(_len(v, rendering) for v in x) + len(sep) * max(len(x) - 1, 0)
    if rendering == TQ:
        return len(json.dumps(x))
    return len(json.dumps(x, ensure_ascii=False, separators=(",", ":")).encode())


def expect(ops, rest, rendering):
    """(UNSUPPORTED, None), (ERROR, the B9_EXC_* bit) or (VALUE, the Python value) of cscript(ops, *rest)"""
    try:
        parsed = parse(ops, len(rest))
    except Unsure:
        return UNSUPPORTED, None
    if parsed is None:
        return ERROR, 0x01
    if not any(code >= LIST_BEGIN for code, _ in parsed):
        return CT.expect(ops, rendering)                   # scalars and strings only: the contract's own rules
    ret, first, kind = run_pass(parsed, rest, rendering, False)
    if ret != 0:
        return (ERROR, ret) if 0 < ret <= CT.EXC_ALL and not ret & (ret - 1) else (UNSUPPORTED, None)
    if first is _Bad or (rendering == ENDPOINT and type(first) is float and not math.isfinite(first)):
        return UNSUPPORTED, None
    if kind == "scalar":
        return VALUE, first                                # a top-level number, bool or None: no writing pass
    value = _py(first)
    if rendering == TQ and not value:
        return VALUE, value                                # falsy: no record bytes, no writing pass
    _, second, _ = run_pass(parsed, rest, rendering, True)
    if second is _Bad or _len(second, rendering) != _len(first, rendering):
        return UNSUPPORTED, None                           # the writing pass broke a rule, or its length differs
    return VALUE, _py(second)


def twin(rendering):
    def cscript(ops, *rest):
        kind, x = expect(ops, list(rest), rendering)
        if kind == ERROR:
            raise CT.exception(x)
        if kind == UNSUPPORTED:
            raise Declined()
        return x
    return cscript
