"""Runs the REFERENCE's own function and endpoint runners with a stub callback URL and freezes the callback each one signs
and posts per task.

    B9_REFERENCE_SDK=<beta9 checkout>/sdk/src python tests/golden/make_ref_callback_runners_golden.py   (from the repo root)

Function runner: the unmodified `invoke_function` (sdk/src/beta9/runner/function.py:236-283), then `complete_task` or
`handle_task_failure` (:285-343), which call the reference's `end_task_and_send_callback` and `send_callback`
(runner/common.py:405-481) with `config.callback_url` set; the function stub hands over each blob as
make_ref_function_full_golden.py's does.
Endpoint runner: an `EndpointManager` built by its own __init__ (a stand-in worker, no gunicorn), its FastAPI app called as
an ASGI application with `POST /` and an X-TASK-ID header, so that `TaskLifecycleMiddleware` -> `middleware.run_task`
(sdk/src/beta9/middleware.py:29-78) wraps the manager's route; the body is what the gateway forwards
(oracle/pyoracle/endpoint.gateway_body), and a body the gateway refuses is its 400 (no task).
Stood in for, in both: the gateway stub (start_task / end_task answer ok; sign_payload records the bytes it is asked to
sign and answers with the oracle's SignPayload), `requests.post` (a recorder that prepares the request as requests does
and keeps the body bytes or the InvalidJSONError; nothing is sent) and `time.sleep` (end_task_and_send_callback's
retry_grpc_call waits 5, 10 and 20 s between attempts; the attempts are counted, not waited for).

Corpus: ref_function_full_golden.json's blobs and `callback_url` values None, "", 0, "http://x", b"http://x", 5, then
bytes results and keys, NaN / inf values and float keys, DEL, 2-, 3- and 4-byte UTF-8, lone surrogates and nested shared
objects; make_ref_endpoint_golden.py's bodies plus the same characters and falsy results as request bodies.
Output: tests/golden/ref_callback_runners_golden.json, checked by tests/test_callback_runners_on_host.py, which rebuilds
the corpus with function_blobs() / endpoint_bodies(). Per task: the runner's status, the bodies sign_payload was asked to
sign (sha256 prefixes for a COMPLETE, a count for an ERROR), what requests.post got ("=" the signed bytes, "R" refused,
"-" not called or raised), the URL, and the exception that escaped the callback, if any; null for a body the gateway
refuses.
"""
import asyncio
import base64
import hashlib
import json
import logging
import os
import sys
import types
from unittest import mock

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
from make_ref_runner_golden import load_reference_runner  # noqa: E402

HANDLERS = ["identity", "crc32", "vadd_f32", "json_sum"]
STUB_URL = "http://callback.invalid/hook"
KEY = b"workspace-signing-key"
TS = 1760000000
TASK_ID = "00000000-0000-4000-8000-000000000000"


def function_calls():
    """(args, kwargs) of the explicit `.remote` calls beyond the function-full golden's blobs"""
    shared = {"k": ["é", 1.5]}
    out = [(("s",), {"callback_url": u}) for u in (None, "", 0, "http://x", b"http://x", 5)]
    vals = [b"x", [1, b""], {b"k": 1}, float("nan"), [float("inf")], {float("-inf"): 1}, {1.5: 1}, {2 ** 63: 1}, 2 ** 63,
            "\x7f", "é", "€", "\U0001F600", "\ud800", "x\ud83dy", [shared, shared, (shared,)], None, "", 0, [], {},
            {None: 1, True: 2, 2.5: 3, "k": [()]}]
    return out + [((v,), {}) for v in vals]


def function_blobs():
    from oracle.pyoracle import funcloop
    g = json.load(open(os.path.join(HERE, "ref_function_full_golden.json")))
    return [base64.b64decode(c["args_pickle"]) for c in g["cases"]] + [funcloop.frame_call(*a, **k) for a, k in function_calls()]


def endpoint_bodies():
    from make_ref_endpoint_golden import bodies
    args = lambda v: b'{"args": [' + v + b']}'                          # noqa: E731
    extra = [args(s) for s in (b'"\x7f"', b'"\xc3\xa9"', b'"\xe2\x82\xac"', b'"\xf0\x9f\x98\x80"', b'"\\ud800"', b'"a\\u0000b"',
                               b'""', b'0', b'[]', b'{}', b'{"values": [1e308, 1e308]}', b'[1, {"a": "\\u00e9", "b": [true, null]}]')]
    extra += [b'{"args": ["x"], "kwargs": {"callback_url": "http://x"}}']
    return bodies() + [b for b in extra if b not in bodies()]


class Recorder:
    """The gateway stub and requests.post of one task: what was signed and posted."""
    def __init__(self, rc):
        self.rc = rc
        self.reset()

    def reset(self):
        self.signed, self.posted, self.url, self.status = [], None, None, None

    # gateway stub
    def start_task(self, req):
        return types.SimpleNamespace(ok=True)

    def end_task(self, req):
        self.status = str(req.task_status)
        return self.rc.EndTaskResponse(ok=True)

    def sign_payload(self, req):
        from oracle.pyoracle import callback as cb
        self.signed.append(bytes(req.payload).decode())
        sig, ts = cb.sign_payload(bytes(req.payload), KEY, TS)
        return self.rc.SignPayloadResponse(ok=True, signature=sig, timestamp=ts)

    # requests.post
    def post(self, url, data=None, json=None, headers=None, **kw):
        import requests
        self.url = url if isinstance(url, str) else repr(url)
        try:
            requests.Request("POST", url, json=json, data=data, headers=headers).prepare()
            self.posted = "="
        except requests.exceptions.InvalidJSONError:
            self.posted = "R"

    def row(self, raised=None):
        """An ERROR's signed body holds the exception text or a traceback (with the runner's file paths): only how many
        bodies were signed is kept for it. A COMPLETE's are kept as sha256 prefixes of their bytes."""
        signed = [body_digest(b.encode()) for b in self.signed] if self.status == "COMPLETE" else len(self.signed)
        return {"status": self.status, "signed": signed, "posted": self.posted or "-", "url": self.url, "raised": raised}


def body_digest(body: bytes) -> str:
    return hashlib.sha256(body).hexdigest()[:24]


def run_function(rc, rf, cf, rec, handler, blobs):
    from oracle.pyoracle import handlers as H
    import beta9.abstractions.function as af
    parent = af.Function.__new__(af.Function)
    parent.stub_id = "stub"; parent.headless = False; parent.handler = "mod:f"
    mod = types.ModuleType("ref_fn_cb_handlers")
    setattr(mod, handler, af._CallableWrapper(getattr(H, handler), parent))
    sys.modules["ref_fn_cb_handlers"] = mod
    rc.config.handler = f"ref_fn_cb_handlers:{handler}"
    rows = []
    for blob in blobs:
        class FnStub:
            def function_get_args(self, req):
                return cf.FunctionGetArgsResponse(ok=True, args=blob)

            def function_set_result(self, req):
                return cf.FunctionSetResultResponse(ok=True)

        ctx = rc.FunctionContext.new(config=rc.config, task_id=TASK_ID, on_start_value=None)
        res = asyncio.run(rf.invoke_function(FnStub(), ctx, TASK_ID))
        rec.reset()
        raised = None
        try:
            if res.exception is None:
                rf.complete_task(rec, res, TASK_ID, "c", "h", 0.0)
            else:
                rf.handle_task_failure(rec, res, TASK_ID, "c", "h")
        except BaseException as e:                                   # (after retry_grpc_call's four attempts)
            raised = type(e).__name__
        rows.append(rec.row(raised))
    return rows


def run_endpoint(rc, re_, rec, handler, bodies):
    from oracle.pyoracle import handlers as H
    from oracle.pyoracle.endpoint import gateway_body
    from oracle.pyoracle.httpserialize import InvalidRequestPayload
    mod = types.ModuleType("ref_ep_cb_handlers")
    setattr(mod, handler, getattr(H, handler))
    sys.modules["ref_ep_cb_handlers"] = mod
    rc.config.handler = f"ref_ep_cb_handlers:{handler}"
    logger = logging.getLogger("ref-callback-runners-golden")
    logger.disabled = True
    mg = re_.EndpointManager(logger, types.SimpleNamespace(notify=lambda: None))
    mg.app.state.gateway_stub = rec
    rows = []
    for b in bodies:
        try:
            forwarded = gateway_body(b)
        except InvalidRequestPayload:
            rows.append(None)                                        # the gateway's 400: no task, no runner
            continue
        rec.reset()
        scope = {"type": "http", "asgi": {"version": "3.0"}, "http_version": "1.1", "method": "POST", "scheme": "http",
                 "path": "/", "raw_path": b"/", "root_path": "", "query_string": b"", "server": ("localhost", 80),
                 "client": ("127.0.0.1", 1), "headers": [(b"x-task-id", TASK_ID.encode()), (b"content-type", b"application/json"),
                                                          (b"content-length", str(len(forwarded)).encode())]}
        sent = []

        async def receive(body=forwarded):
            return {"type": "http.request", "body": body, "more_body": False}

        async def send(msg):
            sent.append(msg)

        raised = None
        try:
            asyncio.run(mg.app(scope, receive, send))
        except BaseException as e:
            raised = type(e).__name__
        rows.append(rec.row(raised))
    return rows


def main():
    from make_ref_endpoint_golden import _EndpointMockFinder
    sys.meta_path.append(_EndpointMockFinder())                     # gunicorn: the endpoint's process model, not installed
    load_reference_runner()
    os.environ["STUB_TYPE"] = "endpoint/deployment"
    import beta9.runner.common as rc
    import beta9.runner.function as rf
    import beta9.clients.function as cf
    import beta9.runner.endpoint as re_
    rc.config.callback_url = STUB_URL
    rc.config.stub_type = "endpoint/deployment"
    rec = Recorder(rc)
    fb, eb = function_blobs(), endpoint_bodies()
    out = {"source": "reference runners: runner/function.py:236-343 (invoke_function, complete_task, handle_task_failure), "
                     "middleware.py:29-78 around runner/endpoint.py's route; runner/common.py:405-481 (send_callback)",
           "stub_url": STUB_URL, "key": KEY.decode(), "ts": TS,
           "function": {"n": len(fb), "handlers": {}}, "endpoint": {"n": len(eb), "handlers": {}}}
    saved_out = sys.stdout
    with mock.patch.object(rc.requests, "post", rec.post), mock.patch.object(rc.time, "sleep", lambda s: None):
        sys.stdout = open(os.devnull, "w")                           # (the runners print progress and tracebacks)
        try:
            for h in HANDLERS:
                out["function"]["handlers"][h] = run_function(rc, rf, cf, rec, h, fb)
                out["endpoint"]["handlers"][h] = run_endpoint(rc, re_, rec, h, eb)
        finally:
            sys.stdout.close()
            sys.stdout = saved_out
    path = os.path.join(HERE, "ref_callback_runners_golden.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
    os.write(2, b"%s %d blobs and %d bodies x %d handlers through the reference runners\n" % (path.encode(), len(fb), len(eb), len(HANDLERS)))


if __name__ == "__main__":
    main()
