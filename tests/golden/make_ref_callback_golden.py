"""Runs the REFERENCE's own runner loop with a stub callback URL and freezes the callback it signs and posts per task.

    B9_REFERENCE_SDK=<beta9 checkout>/sdk/src python tests/golden/make_ref_callback_golden.py   (run from the repo root)

The same harness as make_ref_runner_golden.py: the unmodified `TaskQueueWorker.process_tasks`
(sdk/src/beta9/runner/taskqueue.py:297-404), here with `config.callback_url` set and the reference's own
`send_callback` (runner/common.py:430-481) kept. Two things are stood in for: the gateway stub, whose `sign_payload`
records the bytes it is asked to sign (and answers with the oracle's SignPayload, oracle/pyoracle/callback.py), and
`requests.post`, replaced by a recorder that prepares the request as requests does (`requests.Request(...).prepare()`:
complexjson.dumps(json, allow_nan=False)) and keeps the body bytes or the InvalidJSONError. Nothing is sent.

Corpus: the wires make_ref_retry_golden.py uses (hot_path_golden.json's and the fuzz payloads'), for all four handlers,
then a few explicit payloads: `callback_url` keyword arguments with a URL, "", null and 1, and json_sum totals that
overflow to inf / -inf.
Output: tests/golden/ref_callback_golden.json, checked on every CPU run by tests/test_callback_on_host.py. Per handler,
one letter per task in corpus order (see LETTERS) for its status, whether sign_payload was called, what requests.post
got (the signed bytes, a refusal, nothing) and the URL, plus one sha256 over every signed body (each prefixed by its
length as 8 big-endian bytes) and one over the X-Task-ID / X-Task-Status headers; the explicit tasks are kept whole.

run_reference_worker (make_ref_runner_golden.py) installs its own gateway stub and a no-op callback on the runner
module; it is handed a view of that module which keeps the recording stub and the reference's send_callback instead.
"""
import hashlib
import json
import os
import sys
import struct
from unittest import mock

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from tests.golden.make_ref_retry_golden import corpus_wires  # noqa: E402
from tests.golden.make_ref_runner_golden import HANDLERS, load_reference_runner, run_reference_worker  # noqa: E402

STUB_URL = "http://callback.invalid/hook"
KEY = b"workspace-signing-key"
TS = 1760000000
OVERRIDE_URL = "http://override.invalid/cb"
LETTERS = {"status": {"COMPLETE": "C", "ERROR": "E"}, "signed": "S = sign_payload called, - = not",
           "posted": "= the signed bytes, R = refused (InvalidJSONError), - = nothing (no call, or requests raised first)",
           "url": "S = the stub's URL, O = the override, ? = another value, - = requests.post not called"}


class _KeepCallbackStubs:
    """The runner module as run_reference_worker sees it: every attribute read and write goes to the module, except
    that its assignments of GatewayServiceStub and send_callback are dropped (this file installs its own first)."""
    KEEP = ("GatewayServiceStub", "send_callback")

    def __init__(self, mod):
        object.__setattr__(self, "_mod", mod)

    def __getattr__(self, name):
        return getattr(self._mod, name)

    def __setattr__(self, name, value):
        if name not in self.KEEP:
            setattr(self._mod, name, value)


def explicit_payloads():
    """(payload, task id) pairs beyond the shared corpus: callback_url keyword arguments and non-finite json_sum totals."""
    from oracle.pyoracle import loop
    out = [loop.sdk_put_payload("x", callback_url="http://override.invalid/cb"), loop.sdk_put_payload("x", callback_url=""),
           loop.sdk_put_payload("x", callback_url=None), loop.sdk_put_payload("x", callback_url=1),
           loop.sdk_put_payload(callback_url="http://override.invalid/cb"),
           loop.sdk_put_payload({"values": [1e308, 1e308]}), loop.sdk_put_payload({"values": [-1e308, -1e308]}),
           loop.sdk_put_payload({"values": [1e308, 1e308, -1e308, -1e308]}), loop.sdk_put_payload({"values": []}),
           loop.sdk_put_payload(""), loop.sdk_put_payload("a"), loop.sdk_put_payload("x", "y")]
    return out, [bytes([0xCB, i]) + bytes(14) for i in range(len(out))]


def explicit_wires(handler: str):
    from oracle.pyoracle import loop
    payloads, ids = explicit_payloads()
    return [w.wire for w in loop.run_task_loop(payloads, ids, handler, keep_wire=True) if w.wire is not None]


def run_with_callbacks(rt, rc, handler, wires):
    """-> (done, events): the reference loop over `wires` with the reference's send_callback; events[i] is what the
    callback after task i signed and posted."""
    import requests
    from oracle.pyoracle import callback as cb
    rc.config.callback_url = STUB_URL
    events, completed = {}, [0]
    real_response = rt.TaskQueueCompleteResponse

    def counting_response(*a, **k):              # the harness's task_queue_complete answers with this: count completions
        completed[0] += 1
        return real_response(*a, **k)

    class RecordingGatewayStub:
        def __init__(self, channel=None):
            pass

        def sign_payload(self, req):
            sig, ts = cb.sign_payload(bytes(req.payload), KEY, TS)
            events.setdefault(completed[0] - 1, {})["signed"] = bytes(req.payload)
            return rc.SignPayloadResponse(ok=True, signature=sig, timestamp=ts)

    def post(url, data=None, json=None, headers=None, **kw):
        ev = events.setdefault(completed[0] - 1, {})
        ev["headers"], ev["url"] = dict(headers or {}), url
        try:
            ev["posted"] = requests.Request("POST", url, json=json, data=data, headers=headers).prepare().body
        except requests.exceptions.InvalidJSONError:
            ev["posted"] = "refused"

    saved = rt.GatewayServiceStub, rt.send_callback
    rt.TaskQueueCompleteResponse = counting_response
    rt.GatewayServiceStub, rt.send_callback = RecordingGatewayStub, rc.send_callback
    try:
        with mock.patch.object(rc.requests, "post", post):
            done = run_reference_worker(_KeepCallbackStubs(rt), rc, handler, wires)
    finally:
        rt.TaskQueueCompleteResponse = real_response
        rt.GatewayServiceStub, rt.send_callback = saved
    return done, events


def url_letter(url) -> str:
    return "-" if url is None else "S" if url == STUB_URL else "O" if url == OVERRIDE_URL else "?"


def signed_digest(bodies) -> str:
    """sha256 over the signed bodies in order, each prefixed by its length as 8 big-endian bytes"""
    h = hashlib.sha256()
    for b in bodies:
        h.update(struct.pack(">Q", len(b)) + b)
    return h.hexdigest()


def headers_digest(rows) -> str:
    """sha256 over the "X-Task-ID X-Task-Status" lines of the posted requests, in order"""
    return hashlib.sha256("".join(f"{i} {s}\n" for i, s in rows).encode()).hexdigest()


def main():
    rt, rc = load_reference_runner()
    out = {"source": "reference runner loop (sdk/src/beta9/runner/taskqueue.py:297-404) with config.callback_url set and the "
                     "reference's send_callback (runner/common.py:430-481); sign_payload and requests.post recorded",
           "stub_url": STUB_URL, "key": KEY.decode(), "ts": TS, "letters": LETTERS, "handlers": {}}
    for h in HANDLERS:
        extra = explicit_wires(h)
        wires = corpus_wires(h) + extra
        done, events = run_with_callbacks(rt, rc, h, wires)
        assert len(done) == len(wires), (h, len(done), len(wires))
        rec = {"n": len(wires), "status": "", "signed": "", "posted": "", "url": "", "explicit": []}
        bodies, hdrs = [], []
        for i, (task_id, status, result) in enumerate(done):
            ev = events.get(i, {})
            signed, posted = ev.get("signed"), ev.get("posted")
            assert posted is None or posted == "refused" or posted == signed, (h, i)      # requests posts the signed bytes
            rec["status"] += LETTERS["status"][str(status)]
            rec["signed"] += "-" if signed is None else "S"
            rec["posted"] += "-" if posted is None else "R" if posted == "refused" else "="
            rec["url"] += url_letter(ev.get("url"))
            if signed is not None:
                bodies.append(signed)
            if "headers" in ev:
                hdrs.append((ev["headers"]["X-Task-ID"], ev["headers"]["X-Task-Status"]))
            if i >= len(done) - len(extra):
                rec["explicit"].append([str(status), None if signed is None else signed.decode(), rec["posted"][-1],
                                        None if ev.get("url") is None else str(ev["url"])])
        rec["signed_sha256"], rec["headers_sha256"] = signed_digest(bodies), headers_digest(hdrs)
        out["handlers"][h] = rec
    path = os.path.join(HERE, "ref_callback_golden.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
    print(path, sum(v["n"] for v in out["handlers"].values()), "task executions through the reference runner")


if __name__ == "__main__":
    main()
