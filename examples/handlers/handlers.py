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


TWINS = {"echo_str": echo_str, "crc32_str": crc32_str, "word_count": word_count, "prod": prod}
