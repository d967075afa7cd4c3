"""The Python twins of the example device handlers (handlers.cuh): each is the function a beta9 stub would run. The
tests run them through the reference loops (oracle.pyoracle.loop.run_task_loop, oracle.pyoracle.endpoint.
run_endpoint_request) and compare the device's records with what they produce."""
import zlib


def echo_str(s, /):
    if type(s) is not str:
        raise TypeError("echo_str takes a str")
    return s


def crc32_str(s, /):
    return zlib.crc32(s.encode())


def word_count(s, /):
    return len(s.split())


def prod(xs, /):
    p = 1
    for x in xs:
        if type(x) not in (int, float, bool):
            raise TypeError("prod multiplies numbers")
        p *= x
    return p


def greet(name, greeting="Hello", *, punct="!"):
    return greeting + ", " + name + punct


def join(sep, *parts):
    if type(sep) is not str or any(type(p) is not str for p in parts):
        raise TypeError("join joins strs")
    return sep.join(parts)


def field_sum(rows, *, field):
    if type(field) is not str:
        raise TypeError("field is a str")
    total = 0
    for row in rows:
        if type(row) is not dict:
            raise TypeError("field_sum sums the fields of dicts")
        v = row[field]
        if type(v) not in (int, float, bool):
            raise TypeError("field_sum adds numbers")
        total += v
    return total


def tokens(s, /):
    return s.split()


def grid(s, /):
    return [line.split() for line in s.split("\n")]


def describe(x, /):
    return {"type": type(x).__name__, "value": x}


def pick(d, /, *keys):
    if type(d) is not dict:
        raise TypeError("pick picks from a dict")
    return {k: d[k] for k in keys}


TWINS = {"echo_str": echo_str, "crc32_str": crc32_str, "word_count": word_count, "prod": prod,
         "greet": greet, "join": join, "field_sum": field_sum,
         "tokens": tokens, "grid": grid, "describe": describe, "pick": pick}
