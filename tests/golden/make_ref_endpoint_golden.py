"""Runs the REFERENCE's own endpoint runner over HTTP request bodies under all four handlers and freezes what it answered.

    B9_REFERENCE_SDK=<beta9 checkout>/sdk/src python tests/golden/make_ref_endpoint_golden.py   (from the repo root)

For each body, the gateway's half (pkg/abstractions/endpoint/buffer.go:460-508: SerializeHttpPayload, then
json.Marshal(TaskPayload)) is the oracle's restatement (oracle/pyoracle/endpoint.gateway_body); a body it refuses is the
gateway's 400. What the container does with the forwarded bytes is the unmodified reference: `json.loads` as
`request.json()` does, `EndpointManager._call_function` (sdk/src/beta9/runner/endpoint.py:269-306: the args / kwargs
rules, FunctionHandler.__call__, a raise -> 500 with TaskStatus.Error) and `EndpointManager._create_response`
(:256-267: JSONResponse, a render failure -> 500), with the installed FastAPI / Starlette doing the rendering. The
manager is created without its __init__ (that starts the gunicorn worker machinery); `gunicorn` and `watchdog` are
stood in for by mock modules (not on the data path). The user handlers are oracle/pyoracle/handlers.py, loaded through
the reference's HANDLER=module:func mechanism.

Output: tests/golden/ref_endpoint_golden.json, checked by tests/test_endpoint_on_host.py (oracle and the host build of
endpoint_device.cuh) and tests/test_gpu_endpoint.py (the device)."""
import asyncio
import base64
import importlib.abc
import importlib.machinery
import json
import logging
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, ROOT)
from make_ref_runner_golden import _MockLoader, load_reference_runner  # noqa: E402

HANDLERS = ["identity", "crc32", "vadd_f32", "json_sum"]


class _EndpointMockFinder(importlib.abc.MetaPathFinder):
    """gunicorn: the endpoint module's process model (GunicornApplication / Arbiter), not installed here"""
    def find_spec(self, name, path, target=None):
        if name.split(".")[0] == "gunicorn":
            return importlib.machinery.ModuleSpec(name, _MockLoader(), is_package=True)
        return None


def bodies():
    """The request bodies: test_gpu_parity's HTTP bodies, then the endpoint's rendering and call-rule corners."""
    from tests.test_gpu_parity import _http_bodies
    out = list(_http_bodies())
    args = lambda v: b'{"args": [' + v + b']}'                         # noqa: E731
    for v in (b'""', b'0', b'-0', b'-0.0', b'0.0', b'null', b'false', b'true', b'[]', b'{}', b'[ ]', b'{ }',
              b'1.0', b'1e21', b'1e-7', b'12345678901234567890', b'-12.5e3', b'1E400'):
        out.append(args(v))
    for s in (b'"\xc3\xa9"', b'"\\u00e9"', b'"\xe2\x80\xa8"', b'"\\u2028"', b'"<a&b>"', b'"\\u003c"', b'"\x7f"', b'"\\u007f"',
              b'"\\ud800"', b'"\\udc00x"', b'"\\ud83d\\ude00"', b'"\xf0\x9f\x98\x80"', b'"\xff"', b'"a\xc3"', b'"\xed\xa0\x80"',
              b'"\\"\\\\\\/"', b'"tab\\there"'):
        out.append(args(s))
    out += [args(b'"\\u%04x"' % c) for c in range(0x20)]
    out += [args(b'[1, "a", {"b": null}]'), args(b'{"b": 1, "a": 2, "b": 3}'), args(b'{"z": {"y": [1.5, -0, 2e-7]}, "a": "\xc3\xa9"}'),
            args(b'[[[[[[[[[[[[[[[[[1]]]]]]]]]]]]]]]]]'), args(b'{"k": [true, false, null, 0.1, 100]}')]
    for vals in (b'[1, 2, 3]', b'[1.5, 2.5]', b'[0.0]', b'[-0.0]', b'[0]', b'[]', b'[1, -1]', b'[0.1, 0.2]', b'[1e308, 1e308]',
                 b'[1e308, 1e308, -1e308]', b'[-1e308, -1e308]', b'[9223372036854775807, 1]', b'[true, 2]', b'[1, 2.0]'):
        out.append(args(b'{"values": ' + vals + b'}'))
    for b64 in (b'""', b'"AACAPwAAAEA="', b'"AACAPwAAAEAAAEBAAACAQA=="', b'"AAAA"', b'"!!!!"', b'"AAA="', b'"\\u0041AAA"'):
        out.append(args(b64))
    out += [b'{"args": ["x"], "kwargs": {"k": 1}}', b'{"args": ["cb"], "kwargs": {"callback_url": "http://callback"}}',
            b'{"args": ["x"], "kwargs": {}}', b'{"args": ["x"], "extra": 1}', b'{"args": ["x"], "kwargs": null}', b'{"args": null}',
            b'{"args": ["a", "b"]}', b'{"kwargs": {"s": "x"}}', b'{"s": "x"}']
    seen, uniq = set(), []
    for b in out:
        if b not in seen:
            seen.add(b)
            uniq.append(b)
    return uniq


def main():
    sys.meta_path.append(_EndpointMockFinder())
    os.environ["STUB_TYPE"] = "endpoint/deployment"
    load_reference_runner()
    import beta9.runner.common as rc
    import beta9.runner.endpoint as re_
    from oracle.pyoracle import handlers as H
    from oracle.pyoracle.endpoint import gateway_body
    from oracle.pyoracle.httpserialize import InvalidRequestPayload

    mod = types.ModuleType("ref_ep_handlers")
    for h in HANDLERS:
        setattr(mod, h, getattr(H, h))
    sys.modules["ref_ep_handlers"] = mod
    out = {"source": "reference endpoint runner: runner/endpoint.py:256-306 (_call_function, _create_response)", "cases": []}
    bs = bodies()
    cases = [{"body": base64.b64encode(b).decode(), "results": {}} for b in bs]
    for h in HANDLERS:
        rc.config.handler = f"ref_ep_handlers:{h}"
        mg = re_.EndpointManager.__new__(re_.EndpointManager)
        mg.logger = logging.getLogger("ref-endpoint-golden")
        mg.logger.disabled = True
        mg.handler = rc.FunctionHandler()
        mg.on_start_value = None
        for b, c in zip(bs, cases):
            try:
                forwarded = gateway_body(b)
            except InvalidRequestPayload:
                c["results"][h] = {"status_code": 400, "task_status": None, "body": None}
                continue
            payload = json.loads(forwarded)
            sys.stdout.flush()
            saved, devnull = os.dup(1), os.open(os.devnull, os.O_WRONLY)
            os.dup2(devnull, 1)                                       # (the runner prints a raised handler's traceback)
            try:
                result, error = asyncio.run(mg._call_function(task_id="00000000-0000-4000-8000-000000000000", payload=payload))
            finally:
                os.dup2(saved, 1)
                os.close(saved)
                os.close(devnull)
            status_code = 500 if error else 200
            resp = mg._create_response(body=result, status_code=status_code)
            c["results"][h] = {"status_code": int(resp.status_code), "task_status": "ERROR" if error else "COMPLETE",
                               "body": base64.b64encode(bytes(resp.body)).decode() if resp.status_code == 200 else None}
    out["cases"] = cases
    path = os.path.join(ROOT, "tests", "golden", "ref_endpoint_golden.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
    print(path, len(cases), "bodies x", len(HANDLERS), "handlers through the reference endpoint runner")


if __name__ == "__main__":
    main()
